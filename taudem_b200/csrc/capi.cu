// C ABI of taudem_b200: device-strip level and host-grid level entry points
// (declared in include/taudem_b200.h).  File-level entry points live in tools.cpp.
#include <math.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <string>
#include <vector>

#include "kernels.h"
#include "rowfact.cuh"

namespace td {
unsigned long long g_launches = 0;
static thread_local std::string g_err;
static double g_compute_s = 0.0;

void set_error(const std::string& msg) { g_err = msg; }
int cuda_fail(cudaError_t e, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return (e == cudaErrorMemoryAllocation) ? TD_ERR_ALLOC : TD_ERR_CUDA;
}
void set_compute_seconds(double s) { g_compute_s = s; }
}  // namespace td

using td::Strip;

td_ctx::td_ctx() {
  cudaMalloc(&d_ctr, NCTR * sizeof(unsigned long long));
  cudaMallocHost(&h_ctr, NCTR * sizeof(unsigned long long));
  if (d_ctr) cudaMemset(d_ctr, 0, NCTR * sizeof(unsigned long long));
}
td_ctx::~td_ctx() {
  node.release(); cnt.release(); lev.release(); mk.release(); listA.release(); listB.release(); listC.release();
  tileflags.release(); wsched.release(); rowfact.release(); halo.release(); pend.release();
  if (d_ctr) cudaFree(d_ctr);
  if (h_ctr) cudaFreeHost(h_ctr);
}

namespace {
int check_strip(const td_strip& s) {
  if (s.nx <= 0 || s.ny <= 0 || s.pitch < s.nx || (s.pitch % 32) != 0) { td::set_error("bad strip geometry (pitch must be a multiple of 32 and >= nx)"); return TD_ERR_ARG; }
  return TD_OK;
}
int need_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) { td::set_error(std::string("no usable CUDA device: ") + cudaGetErrorString(e)); return TD_ERR_CUDA; }
  return TD_OK;
}
// TAUDEM_B200_TRACE=1: wall-clock marks of the host-grid level calls on stderr (epoch seconds, comparable across processes)
void trace_mark(const char* what) {
  static const bool on = getenv("TAUDEM_B200_TRACE") != nullptr;
  if (!on) return;
  timespec ts; clock_gettime(CLOCK_REALTIME, &ts);
  fprintf(stderr, "[td trace] %.3f %s\n", (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec, what);
}
td_ctx* default_ctx() {
  static td_ctx* c = nullptr;
  if (!c) c = new td_ctx();
  return c;
}
}  // namespace

extern "C" {

const char* td_version(void) { return "5.4.0-b200"; }
const char* td_last_error(void) { return td::g_err.c_str(); }
// starts the CUDA context (file-level tools call it on a helper thread while they read their inputs)
int td_warmup(void) {
  trace_mark("warmup: start");
  const cudaError_t e = cudaFree(0);
  trace_mark("warmup: context ready");
  return e == cudaSuccess ? TD_OK : TD_ERR_CUDA;
}
int td_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }
int td_set_device(int dev) { TD_CUDA(cudaSetDevice(dev)); return TD_OK; }
unsigned long long td_launch_count(void) { return td::g_launches; }
void td_reset_launch_count(void) { td::g_launches = 0; }
double td_last_compute_seconds(void) { return td::g_compute_s; }
int td_pitch_for(int nx) { return (nx + 31) / 32 * 32; }
unsigned long long td_ctx_counter(td_ctx* ctx, int i) {
  unsigned long long v = 0;
  if (!ctx || i < 0 || i >= td_ctx::NCTR) return 0;
  cudaDeviceSynchronize();
  cudaMemcpy(&v, ctx->d_ctr + i, sizeof v, cudaMemcpyDeviceToHost);
  return v;
}


td_ctx* td_ctx_create(void) {
  if (need_device() != TD_OK) return nullptr;
  td_ctx* c = new td_ctx();
  if (!c->d_ctr || !c->h_ctr) { delete c; td::set_error("context allocation failed"); return nullptr; }
  return c;
}
void td_ctx_destroy(td_ctx* c) { delete c; }

// ------------------------------------------------------------------ device-strip level
int td_gen_dem_dev(float* dem, td_strip s, int row0_global, int total_ny, unsigned seed, float hurst, float tilt, void* stream) {
  if (int rc = check_strip(s)) return rc;
  TD_CUDA(td::launch_gen_dem(dem, Strip(s), row0_global, total_ny, seed, hurst, tilt, (cudaStream_t)stream));
  return TD_OK;
}
int td_gen_weights_dev(float* w, td_strip s, int row0_global, unsigned seed, void* stream) {
  if (int rc = check_strip(s)) return rc;
  TD_CUDA(td::launch_gen_w(w, Strip(s), row0_global, seed, (cudaStream_t)stream));
  return TD_OK;
}

int td_flood_init_dev(td_ctx* ctx, const float* dem, const int16_t* depmask, float* planchon, td_strip s, float dem_nodata,
                      int is_4Point, void* stream) {
  (void)ctx;
  if (int rc = check_strip(s)) return rc;
  return td::fill_init(dem, depmask, planchon, Strip(s), dem_nodata, is_4Point, (cudaStream_t)stream);
}
int td_flood_relax_dev(td_ctx* ctx, const float* dem, float* planchon, td_strip s, int is_4Point, int* changed_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  int ch = 0;
  int rc = td::fill_relax(ctx, dem, planchon, Strip(s), is_4Point, &ch, (cudaStream_t)stream);
  if (changed_out) *changed_out = ch;
  return rc;
}

// after an exchange of the halo rows: only the tiles next to them are queued to start with
int td_flood_relax_edges_dev(td_ctx* ctx, const float* dem, float* planchon, td_strip s, int is_4Point, int* changed_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  int ch = 0;
  int rc = td::fill_relax(ctx, dem, planchon, Strip(s), is_4Point, &ch, (cudaStream_t)stream, true);
  if (changed_out) *changed_out = ch;
  return rc;
}

int td_d8_slopes_dev(td_ctx* ctx, const float* fel, int16_t* p, float* sd8, td_strip s, float fel_nodata, const double* dxc,
                     const double* dyc, long long* nflat_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  TD_CUDA(cudaMemsetAsync(ctx->d_ctr + 8, 0, sizeof(unsigned long long), st));
  TD_CUDA(ctx->rowfact.ensure(sizeof(td::RowFact) * (size_t)s.ny));
  td::launch_row_factors(dxc, dyc, nullptr, nullptr, ctx->rowfact.as<td::RowFact>(), s.ny, st);
  if (int rc = td::launch_d8_stencil(fel, p, sd8, ctx->rowfact.as<td::RowFact>(), Strip(s), fel_nodata, ctx->d_ctr + 8, st)) return rc;
  if (nflat_out) {
    TD_CUDA(cudaMemcpyAsync(ctx->h_ctr + 8, ctx->d_ctr + 8, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    TD_CUDA(cudaStreamSynchronize(st));
    *nflat_out = (long long)ctx->h_ctr[8];
  }
  return TD_OK;
}
int td_d8_flats_dev(td_ctx* ctx, float* fel, int16_t* p, td_strip s, const double* dxc, const double* dyc, long long* nflat_left,
                    void* stream) {
  if (int rc = check_strip(s)) return rc;
  long long left = 0;
  int rc = td::resolve_flats_d8(ctx, fel, p, Strip(s), dxc, dyc, &left, nullptr, (cudaStream_t)stream);
  if (nflat_left) *nflat_left = left;
  return rc;
}
int td_d8_flats_strip_dev(td_ctx* ctx, float* fel, int16_t* p, td_strip s, const double* dxc, const double* dyc, long long* nflat_left,
                          const td_strip_comm* comm, void* stream) {
  if (int rc = check_strip(s)) return rc;
  long long left = 0;
  int rc = td::resolve_flats_d8(ctx, fel, p, Strip(s), dxc, dyc, &left, comm, (cudaStream_t)stream);
  if (nflat_left) *nflat_left = left;
  return rc;
}

// per-row atan2 tables are evaluated on the host (glibc), like the reference's prop()/VSLOPE do
static int upload_theta_from_host(td_ctx* ctx, const double* dx, const double* dy, int ny, td_ctx::Buf& buf, cudaStream_t st) {
  // [0, ny) atan2(dy, dx), [ny, 2 ny) atan2(dx, dy), then the angle of the row above and of the row below the strip (theta_of_row)
  std::vector<double> th(2 * (size_t)ny + 2);
  for (int j = 0; j < ny; j++) {
    // (projected rasters: every row has the same cell size — two atan2 calls instead of 2 ny on the critical path of every call)
    if (j > 0 && dx[j] == dx[j - 1] && dy[j] == dy[j - 1]) { th[j] = th[j - 1]; th[ny + j] = th[ny + j - 1]; }
    else { th[j] = atan2(dy[j], dx[j]); th[ny + j] = atan2(dx[j], dy[j]); }
  }
  th[2 * (size_t)ny] = ctx->halo_dx[0] > 0. && ctx->halo_dy[0] > 0. ? atan2(ctx->halo_dy[0], ctx->halo_dx[0]) : th[0];
  th[2 * (size_t)ny + 1] = ctx->halo_dx[1] > 0. && ctx->halo_dy[1] > 0. ? atan2(ctx->halo_dy[1], ctx->halo_dx[1]) : th[ny - 1];
  TD_CUDA(buf.ensure(sizeof(double) * th.size()));
  TD_CUDA(cudaMemcpyAsync(buf.p, th.data(), sizeof(double) * th.size(), cudaMemcpyHostToDevice, st));
  TD_CUDA(cudaStreamSynchronize(st));
  // one prop() table for the whole strip when every row (the neighbours' edge rows included) has the same angle (projected rasters)
  bool uni = th[2 * (size_t)ny] == th[0] && th[2 * (size_t)ny + 1] == th[0];
  for (int j = 1; j < ny && uni; j++) uni = th[j] == th[0] && dx[j] == dx[0];
  td::make_prop_row(th[0], uni, &ctx->prop);
  ctx->dx0 = dx[0];
  return TD_OK;
}
static int upload_theta(td_ctx* ctx, const double* d_dxc, const double* d_dyc, int ny, td_ctx::Buf& buf, cudaStream_t st) {
  std::vector<double> dx(ny), dy(ny);
  TD_CUDA(cudaMemcpyAsync(dx.data(), d_dxc, sizeof(double) * ny, cudaMemcpyDeviceToHost, st));
  TD_CUDA(cudaMemcpyAsync(dy.data(), d_dyc, sizeof(double) * ny, cudaMemcpyDeviceToHost, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return upload_theta_from_host(ctx, dx.data(), dy.data(), ny, buf, st);
}

void td_set_halo_cell_sizes_dev(td_ctx* ctx, double dx_top, double dy_top, double dx_bot, double dy_bot) {
  if (!ctx) return;
  ctx->halo_dx[0] = dx_top; ctx->halo_dy[0] = dy_top; ctx->halo_dx[1] = dx_bot; ctx->halo_dy[1] = dy_bot;
}
int td_dinf_slopes_dev(td_ctx* ctx, const float* fel, float* ang, float* slp, td_strip s, float fel_nodata, const double* dxc,
                       const double* dyc, long long* nflat_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = upload_theta(ctx, dxc, dyc, s.ny, ctx->theta, st)) return rc;
  const double* thA = ctx->theta.as<double>();
  TD_CUDA(cudaMemsetAsync(ctx->d_ctr + 8, 0, sizeof(unsigned long long), st));
  TD_CUDA(ctx->rowfact.ensure(sizeof(td::RowFact) * (size_t)s.ny));
  td::launch_row_factors(dxc, dyc, thA, thA + s.ny, ctx->rowfact.as<td::RowFact>(), s.ny, st);
  if (int rc = td::launch_dinf_stencil(fel, ang, slp, ctx->rowfact.as<td::RowFact>(), Strip(s), fel_nodata, ctx->d_ctr + 8, st)) return rc;
  if (nflat_out) {
    TD_CUDA(cudaMemcpyAsync(ctx->h_ctr + 8, ctx->d_ctr + 8, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    TD_CUDA(cudaStreamSynchronize(st));
    *nflat_out = (long long)ctx->h_ctr[8];
  }
  return TD_OK;
}
int td_dinf_flats_dev(td_ctx* ctx, float* fel, float* ang, td_strip s, const double* dxc, const double* dyc, long long* nflat_left,
                      void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = upload_theta(ctx, dxc, dyc, s.ny, ctx->theta, st)) return rc;
  const double* thA = ctx->theta.as<double>();
  long long left = 0;
  int rc = td::resolve_flats_dinf(ctx, fel, ang, Strip(s), dxc, dyc, thA, thA + s.ny, &left, nullptr, st);
  if (nflat_left) *nflat_left = left;
  return rc;
}
int td_dinf_flats_strip_dev(td_ctx* ctx, float* fel, float* ang, td_strip s, const double* dxc, const double* dyc, long long* nflat_left,
                            const td_strip_comm* comm, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = upload_theta(ctx, dxc, dyc, s.ny, ctx->theta, st)) return rc;
  const double* thA = ctx->theta.as<double>();
  long long left = 0;
  int rc = td::resolve_flats_dinf(ctx, fel, ang, Strip(s), dxc, dyc, thA, thA + s.ny, &left, comm, st);
  if (nflat_left) *nflat_left = left;
  return rc;
}

static int ensure_dep_state(td_ctx* ctx, const Strip& s, cudaStream_t st) {
  const size_t n = (size_t)s.cells();
  TD_CUDA(ctx->node.ensure(n * 2));
  TD_CUDA(ctx->cnt.ensure((n + 3) / 4 * 4));
  TD_CUDA(ctx->halo.ensure(sizeof(int) * 2 * (size_t)s.pitch));
  TD_CUDA(td::zero_words(ctx->halo.p, sizeof(int) * 2 * (size_t)s.pitch, st));
  return TD_OK;
}

int td_aread8_deps_dev(td_ctx* ctx, const int16_t* p, float* ad8, td_strip s, int16_t p_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = ensure_dep_state(ctx, Strip(s), st)) return rc;
  ctx->sweep_dinf = 0;
  TD_CUDA(td::launch_deps_d8(p, ctx->node.as<unsigned short>(), ctx->cnt.as<unsigned char>(), ad8, Strip(s), p_nodata, st));
  return TD_OK;
}
int td_aread8_sweep_dev(td_ctx* ctx, const float* w, float* ad8, td_strip s, float w_nodata, int usew, int contcheck, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (int rc = td::wsweep_begin(ctx, Strip(s), (cudaStream_t)stream)) return rc;
  return td::wsweep_run(ctx, false, ad8, w, nullptr, Strip(s), w_nodata, usew, contcheck, nullptr, nullptr, ctx->halo.as<int>(), (cudaStream_t)stream);
}

// (theta_ready: the caller has uploaded the row tables of this strip already — upload_theta_from_host — so that no small copy
//  of this call queues behind a raster that is travelling on another stream)
static int area_deps(td_ctx* ctx, const float* ang, float* sca, td_strip s, float ang_nodata, const double* dxc, const double* dyc,
                     bool theta_ready, void* stream, float area_init = -1.0f) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = ensure_dep_state(ctx, Strip(s), st)) return rc;
  if (!theta_ready) { if (int rc = upload_theta(ctx, dxc, dyc, s.ny, ctx->theta, st)) return rc; }
  ctx->sweep_dinf = 1;
  TD_CUDA(td::launch_deps_dinf(ang, ctx->node.as<unsigned short>(), ctx->cnt.as<unsigned char>(), sca, Strip(s), ang_nodata,
                               ctx->theta.as<double>(), st, area_init));
  return TD_OK;
}
int td_area_deps_dev(td_ctx* ctx, const float* ang, float* sca, td_strip s, float ang_nodata, const double* dxc, const double* dyc,
                     void* stream) {
  return area_deps(ctx, ang, sca, s, ang_nodata, dxc, dyc, false, stream);
}
int td_area_sweep_dev(td_ctx* ctx, const float* ang, const float* w, float* sca, td_strip s, int usew, int contcheck,
                      const double* dxc, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const Strip ss(s);
  if (int rc = td::wsweep_begin(ctx, ss, st)) return rc;
  return td::wsweep_run(ctx, true, sca, w, ang, ss, 0.f, usew, contcheck, ctx->theta.as<double>(), dxc, ctx->halo.as<int>(), st);
}

// aread8 / areadinf -o: between *_deps_dev and *_sweep_dev, restricts the dependency state to the cells upstream of the
// outlets (grid coordinates, row 0 = the strip's first owned row; host arrays).  Single strip.
int td_sweep_restrict_dev(td_ctx* ctx, td_strip s, const int* cols, const int* rows, int nout, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (nout < 0 || (nout > 0 && (!cols || !rows))) { td::set_error("td_sweep_restrict_dev: bad arguments"); return TD_ERR_ARG; }
  return td::sweep_restrict_upstream(ctx, Strip(s), cols, rows, nout, (cudaStream_t)stream);
}

// The same over row strips, in rounds like the sweeps: seeds = the outlets of this strip (first round) + the requests the
// neighbour strips recorded for my first / last row (in_top / in_bot, device, pitch ints, NULL = none); req_out (device,
// 2 x pitch ints) receives my requests to them; repeat until nobody requests anything, then one call with finish = 1
// (src/commonLib.cpp:300-375 does this exchange with bufferAbove / bufferBelow and transferPack).
int td_sweep_restrict_round_dev(td_ctx* ctx, td_strip s, const int* cols, const int* rows, int nout, const int* in_top, const int* in_bot,
                                int* req_out, int finish, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if ((nout > 0 && (!cols || !rows)) || !req_out) { td::set_error("td_sweep_restrict_round_dev: bad arguments"); return TD_ERR_ARG; }
  return td::sweep_restrict_round(ctx, Strip(s), cols, rows, nout, in_top, in_bot, req_out, finish, (cudaStream_t)stream);
}

// ---- multi-strip sweeps: begin (queue all tiles) / run (until locally drained; crossings into the
// neighbour strips are counted in halo_out[0..pitch) = row above, [pitch..2*pitch) = row below) /
// apply (decrements received from the neighbours for my first / last row)
int td_sweep_begin_dev(td_ctx* ctx, td_strip s, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_begin(ctx, Strip(s), (cudaStream_t)stream);
}
int td_sweep_apply_halo_dev(td_ctx* ctx, td_strip s, const int* dec_top, const int* dec_bot, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_apply_halo(ctx, Strip(s), dec_top, dec_bot, (cudaStream_t)stream);
}
int td_aread8_sweep_run_dev(td_ctx* ctx, const float* w, float* ad8, td_strip s, float w_nodata, int usew, int contcheck, int* halo_out,
                            void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_run(ctx, false, ad8, w, nullptr, Strip(s), w_nodata, usew, contcheck, nullptr, nullptr, halo_out, (cudaStream_t)stream);
}
int td_area_sweep_run_dev(td_ctx* ctx, const float* ang, const float* w, float* sca, td_strip s, int usew, int contcheck, const double* dxc,
                          int* halo_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_run(ctx, true, sca, w, ang, Strip(s), 0.f, usew, contcheck, ctx->theta.as<double>(), dxc, halo_out, (cudaStream_t)stream);
}

}  // extern "C"
namespace td {
// gridnet's cell-to-cell distances of rows 0 .. ny - 1: dist[row][k - 1] = sqrt(dxc^2 d1[k]^2 + dyc^2 d2[k]^2) as float (src/gridnet.cpp:190-200)
void gridnet_dist_table(const double* dxc, const double* dyc, int ny, float* dist) {
  static const int d1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1}, d2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};
  for (int m = 0; m < ny; ++m)
    for (int k = 1; k <= 8; ++k) dist[(size_t)m * 8 + k - 1] = (float)sqrt(dxc[m] * dxc[m] * d1[k] * d1[k] + dyc[m] * dyc[m] * d2[k] * d2[k]);
}
}  // namespace td
extern "C" {

// ---- the five sibling sweep tools on row strips: the same protocol (deps, begin, rounds of run + apply_halo, or peer mode)
int td_d8flowpathextremeup_deps_dev(td_ctx* ctx, const int16_t* p, float* ssa, td_strip s, int16_t p_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = ensure_dep_state(ctx, Strip(s), st)) return rc;
  ctx->sweep_dinf = 0;
  TD_CUDA(td::launch_deps_d8(p, ctx->node.as<unsigned short>(), ctx->cnt.as<unsigned char>(), ssa, Strip(s), p_nodata, st, TD_MISSINGFLOAT));
  return TD_OK;
}
int td_d8flowpathextremeup_sweep_run_dev(td_ctx* ctx, const float* sa, float* ssa, td_strip s, int usemax, int contcheck, int* halo_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_run(ctx, false, ssa, sa, nullptr, Strip(s), 0.f, 1, contcheck, nullptr, nullptr, halo_out, (cudaStream_t)stream, usemax ? 1 : 2);
}
int td_dinfdecayaccum_deps_dev(td_ctx* ctx, const float* ang, float* dsca, td_strip s, float ang_nodata, const double* dxc, const double* dyc, void* stream) {
  return area_deps(ctx, ang, dsca, s, ang_nodata, dxc, dyc, false, stream, TD_MISSINGFLOAT);
}
int td_dinfdecayaccum_sweep_run_dev(td_ctx* ctx, const float* ang, const float* dm, const float* w, float* dsca, td_strip s, float dm_nodata, int contcheck,
                                    const double* dxc, int* halo_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_run(ctx, true, dsca, w, ang, Strip(s), 0.f, w != nullptr, contcheck, ctx->theta.as<double>(), dxc, halo_out, (cudaStream_t)stream, 3,
                        dm, dm_nodata);
}
int td_dinfconclimaccum_deps_dev(td_ctx* ctx, const float* ang, float* ctpt, td_strip s, float ang_nodata, const double* dxc, const double* dyc, void* stream) {
  return area_deps(ctx, ang, ctpt, s, ang_nodata, dxc, dyc, false, stream, TD_MISSINGFLOAT);
}
int td_dinfconclimaccum_sweep_run_dev(td_ctx* ctx, const float* ang, const float* dm, const float* q, const int16_t* dg, float* ctpt, td_strip s, float dm_nodata,
                                      float q_nodata, float csol, int contcheck, const double* dxc, int* halo_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  td::SweepExtra x; x.dg = dg; x.csol = csol;
  return td::wsweep_run(ctx, true, ctpt, q, ang, Strip(s), q_nodata, 1, contcheck, ctx->theta.as<double>(), dxc, halo_out, (cudaStream_t)stream, 7, dm,
                        dm_nodata, nullptr, &x);
}
int td_dinftranslimaccum_deps_dev(td_ctx* ctx, const float* ang, float* tla, float* tdep, float* ctpt, td_strip s, float ang_nodata, const double* dxc,
                                  const double* dyc, void* stream) {
  if (int rc = area_deps(ctx, ang, tla, s, ang_nodata, dxc, dyc, false, stream, TD_MISSINGFLOAT)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  TD_CUDA(td::fill_floats(tdep, Strip(s), TD_MISSINGFLOAT, st));                 // cells that are never evaluated stay nodata (src/DinfTransLimAccum.cpp:198-204)
  if (ctpt) TD_CUDA(td::fill_floats(ctpt, Strip(s), TD_MISSINGFLOAT, st));
  return TD_OK;
}
int td_dinftranslimaccum_sweep_run_dev(td_ctx* ctx, const float* ang, const float* tsup, const float* tc, const float* cs, float* tla, float* tdep, float* ctpt,
                                       td_strip s, float tsup_nodata, float tc_nodata, float cs_nodata, int contcheck, const double* dxc, int* halo_out,
                                       void* stream) {
  if (int rc = check_strip(s)) return rc;
  if ((cs != nullptr) != (ctpt != nullptr)) { td::set_error("td_dinftranslimaccum_sweep_run_dev: the concentration input and output come together"); return TD_ERR_ARG; }
  td::SweepExtra x; x.cin = cs; x.cin_nodata = cs_nodata; x.out2 = tdep; x.out3 = ctpt;
  return td::wsweep_run(ctx, true, tla, tsup, ang, Strip(s), tsup_nodata, 1, contcheck, ctx->theta.as<double>(), dxc, halo_out, (cudaStream_t)stream,
                        cs ? 9 : 8, tc, tc_nodata, nullptr, &x);
}
int td_gridnet_mask_dev(td_ctx*, const int32_t* mask, float* ok, td_strip s, int thresh, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::launch_mask_ok(mask, ok, Strip(s), thresh, (cudaStream_t)stream);
}
int td_gridnet_deps_dev(td_ctx* ctx, const int16_t* p, float* out, td_strip s, int16_t p_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = ensure_dep_state(ctx, Strip(s), st)) return rc;
  ctx->sweep_dinf = 0;
  TD_CUDA(td::launch_deps_d8(p, ctx->node.as<unsigned short>(), ctx->cnt.as<unsigned char>(), out, Strip(s), p_nodata, st, -1.0f));
  TD_CUDA(td::launch_halo_codes_d8(p, ctx->node.as<unsigned short>(), Strip(s), p_nodata, st));
  return TD_OK;
}
int td_gridnet_sweep_run_dev(td_ctx* ctx, int which, const float* ok, const float* dist, float* out, td_strip s, int outlets, int* halo_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (which < 0 || which > 2 || !dist) { td::set_error("td_gridnet_sweep_run_dev: which = 0, 1 or 2, and the distance table is required"); return TD_ERR_ARG; }
  // cells outside the mask: not evaluated — plen / tlen stay nodata; the Strahler order keeps what the start gave it: 1 if upstream of
  // an outlet (src/gridnet.cpp:296), nodata otherwise
  const float skip = (which == 2 && outlets) ? 1.0f : -1.0f;
  return td::wsweep_run(ctx, false, out, nullptr, nullptr, Strip(s), skip, 0, 0, nullptr, nullptr, halo_out, (cudaStream_t)stream, 4 + which, ok, 0.f, dist);
}
int td_gridnet_order_dev(td_ctx* ctx, const float* order, const int16_t* p, const float* ok, int16_t* gord, td_strip s, int16_t p_nodata, int outlets,
                         void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::launch_gord_finish(order, p, ok, ctx->node.as<unsigned short>(), gord, Strip(s), p_nodata, outlets ? 1 : 0, (cudaStream_t)stream);
}

// ---- peer mode of the partitioned sweeps: neighbours' counts / tile queues / halo buffers mapped over
// NVLink with CUDA IPC; the sweep kernel then delivers across GPUs itself and no exchange rounds exist.
int td_sweep_peer_export_dev(td_ctx* ctx, td_strip s, int dinf, unsigned char* handles_5x64, int* meta_8, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::sweep_peer_export(ctx, Strip(s), dinf, handles_5x64, meta_8, (cudaStream_t)stream);
}
int td_sweep_peer_connect_dev(td_ctx* ctx, int which, const unsigned char* handles_5x64, const int* meta_8) {
  return td::sweep_peer_connect(ctx, which, handles_5x64, meta_8);
}
int td_sweep_peer_begin_dev(td_ctx* ctx, td_strip s, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::sweep_peer_begin(ctx, Strip(s), (cudaStream_t)stream);
}
void td_sweep_peer_off_dev(td_ctx* ctx) { td::sweep_peer_off(ctx); }

}  // extern "C"

// ------------------------------------------------------------------ host-grid level
namespace {
struct Timer {
  cudaEvent_t a, b;
  Timer() { cudaEventCreate(&a); cudaEventCreate(&b); }
  ~Timer() { cudaEventDestroy(a); cudaEventDestroy(b); }
  void start(cudaStream_t st) { cudaEventRecord(a, st); }
  double stop(cudaStream_t st) { cudaEventRecord(b, st); cudaEventSynchronize(b); float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms * 1e-3; }
};
// host dense (nx) <-> device strip rows 1..ny (pitch)
template <typename T> cudaError_t h2d(T* dst, const T* src, const td_strip& s, cudaStream_t st) {
  if (s.pitch == s.nx) {
    // one contiguous block, sent in 64 MiB pieces
    const size_t total = (size_t)s.nx * s.ny * sizeof(T), piece = (size_t)64 << 20;
    for (size_t off = 0; off < total; off += piece) {
      const cudaError_t e = cudaMemcpyAsync((char*)(dst + s.pitch) + off, (const char*)src + off, std::min(piece, total - off), cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  }
  return cudaMemcpy2DAsync(dst + s.pitch, (size_t)s.pitch * sizeof(T), src, (size_t)s.nx * sizeof(T), (size_t)s.nx * sizeof(T), s.ny,
                           cudaMemcpyHostToDevice, st);
}
template <typename T> cudaError_t d2h(T* dst, const T* src, const td_strip& s, cudaStream_t st) {
  if (s.pitch == s.nx) return cudaMemcpyAsync(dst, src + s.pitch, (size_t)s.nx * s.ny * sizeof(T), cudaMemcpyDeviceToHost, st);
  return cudaMemcpy2DAsync(dst, (size_t)s.nx * sizeof(T), src + s.pitch, (size_t)s.pitch * sizeof(T), (size_t)s.nx * sizeof(T), s.ny,
                           cudaMemcpyDeviceToHost, st);
}
td_strip host_strip(int nx, int ny) { td_strip s; s.nx = nx; s.ny = ny; s.pitch = td_pitch_for(nx); s.has_top = 0; s.has_bot = 0; return s; }

int upload_rows(td_ctx* ctx, const double* dxc, const double* dyc, int ny, const double** d_dxc, const double** d_dyc, cudaStream_t st) {
  TD_CUDA(ctx->rows.ensure(sizeof(double) * 2 * (size_t)ny));
  double* d = ctx->rows.as<double>();
  TD_CUDA(cudaMemcpyAsync(d, dxc, sizeof(double) * ny, cudaMemcpyHostToDevice, st));
  TD_CUDA(cudaMemcpyAsync(d + ny, dyc, sizeof(double) * ny, cudaMemcpyHostToDevice, st));
  *d_dxc = d; *d_dyc = d + ny;
  return TD_OK;
}
}  // namespace

extern "C" {

int td_flood_host(const float* dem, float* fel, const int16_t* depmask, int nx, int ny, float dem_nodata, int is_4Point) {
  if (int rc = need_device()) return rc;
  if (!dem || !fel || nx <= 0 || ny <= 0) { td::set_error("td_flood_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4));
  float* d_dem = ctx->io[0].as<float>(); float* d_w = ctx->io[1].as<float>();
  int16_t* d_mask = nullptr;
  TD_CUDA(h2d(d_dem, dem, s, st));
  if (depmask) { TD_CUDA(ctx->io[2].ensure(n * 2)); d_mask = ctx->io[2].as<int16_t>(); TD_CUDA(h2d(d_mask, depmask, s, st)); }
  Timer t; t.start(st);
  if (int rc = td_flood_init_dev(ctx, d_dem, d_mask, d_w, s, dem_nodata, is_4Point, st)) return rc;
  int changed = 0;
  if (int rc = td_flood_relax_dev(ctx, d_dem, d_w, s, is_4Point, &changed, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(fel, d_w, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

int td_setdird8_host(const float* fel, int16_t* p, float* sd8, int nx, int ny, float fel_nodata, const double* dxc, const double* dyc) {
  if (int rc = need_device()) return rc;
  if (!fel || !p || !sd8 || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_setdird8_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 2));
  float* d_fel = ctx->io[0].as<float>(); float* d_sl = ctx->io[1].as<float>(); int16_t* d_p = ctx->io[2].as<int16_t>();
  const double *d_dx, *d_dy;
  if (int rc = upload_rows(ctx, dxc, dyc, ny, &d_dx, &d_dy, st)) return rc;
  TD_CUDA(h2d(d_fel, fel, s, st));
  Timer t; t.start(st);
  long long nflat = 0;
  if (int rc = td_d8_slopes_dev(ctx, d_fel, d_p, d_sl, s, fel_nodata, d_dx, d_dy, &nflat, st)) return rc;
  // the slope raster is final before flats are resolved (src/d8.cpp:282-288)
  if (nflat > 0) { long long left = 0; if (int rc = td_d8_flats_dev(ctx, d_fel, d_p, s, d_dx, d_dy, &left, st)) return rc; }
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(p, d_p, s, st));
  TD_CUDA(d2h(sd8, d_sl, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

int td_setdir_host(const float* fel, float* ang, float* slp, int nx, int ny, float fel_nodata, const double* dxc, const double* dyc) {
  if (int rc = need_device()) return rc;
  if (!fel || !ang || !slp || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_setdir_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 4));
  float* d_fel = ctx->io[0].as<float>(); float* d_sl = ctx->io[1].as<float>(); float* d_ang = ctx->io[2].as<float>();
  const double *d_dx, *d_dy;
  if (int rc = upload_rows(ctx, dxc, dyc, ny, &d_dx, &d_dy, st)) return rc;
  TD_CUDA(h2d(d_fel, fel, s, st));
  Timer t; t.start(st);
  long long nflat = 0;
  if (int rc = td_dinf_slopes_dev(ctx, d_fel, d_ang, d_sl, s, fel_nodata, d_dx, d_dy, &nflat, st)) return rc;
  if (nflat > 0) { long long left = 0; if (int rc = td_dinf_flats_dev(ctx, d_fel, d_ang, s, d_dx, d_dy, &left, st)) return rc; }
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(ang, d_ang, s, st));
  TD_CUDA(d2h(slp, d_sl, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

int td_aread8_host(const int16_t* p, const float* w, float* ad8, int nx, int ny, int16_t p_nodata, float w_nodata, int contcheck) {
  return td_aread8_outlets_host(p, w, ad8, nx, ny, p_nodata, w_nodata, contcheck, nullptr, nullptr, -1);
}

// nout < 0: no outlets (the whole grid); nout >= 0: only the cells upstream of the outlets (src/aread8.cpp -o)
int td_aread8_outlets_host(const int16_t* p, const float* w, float* ad8, int nx, int ny, int16_t p_nodata, float w_nodata, int contcheck,
                           const int* outlet_cols, const int* outlet_rows, int nout) {
  trace_mark("aread8_host: enter");
  if (int rc = need_device()) return rc;
  if (!p || !ad8 || nx <= 0 || ny <= 0) { td::set_error("td_aread8_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  trace_mark("aread8_host: device ready");
  TD_CUDA(ctx->io[0].ensure(n * 2)); TD_CUDA(ctx->io[1].ensure(n * 4));
  int16_t* d_p = ctx->io[0].as<int16_t>(); float* d_a = ctx->io[1].as<float>(); float* d_w = nullptr;
  trace_mark("aread8_host: buffers allocated");
  TD_CUDA(h2d(d_p, p, s, st));
  if (w) { TD_CUDA(ctx->io[2].ensure(n * 4)); d_w = ctx->io[2].as<float>(); TD_CUDA(h2d(d_w, w, s, st)); }
  if (getenv("TAUDEM_B200_TRACE")) { cudaStreamSynchronize(st); trace_mark("aread8_host: inputs on the device"); }
  Timer t; t.start(st);
  if (int rc = td_aread8_deps_dev(ctx, d_p, d_a, s, p_nodata, st)) return rc;
  if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
  if (int rc = td_aread8_sweep_dev(ctx, d_w, d_a, s, w_nodata, w != nullptr, contcheck, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  trace_mark("aread8_host: computed");
  TD_CUDA(d2h(ad8, d_a, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  trace_mark("aread8_host: result on the host");
  return TD_OK;
}

// ---- d8flowpathextremeup (src/D8flowpathextremeup.cpp:58-285): the D8 dependency stencil and sweep with the extreme-value
// algebra — each cell gets the largest (usemax) / smallest value of `sa` on the flow paths that end in it; nodata = MISSINGFLOAT.
int td_d8flowpathextremeup_host(const int16_t* p, const float* sa, float* ssa, int nx, int ny, int16_t p_nodata, int usemax, int contcheck,
                                const int* outlet_cols, const int* outlet_rows, int nout) {
  if (int rc = need_device()) return rc;
  if (!p || !sa || !ssa || nx <= 0 || ny <= 0) { td::set_error("td_d8flowpathextremeup_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 2)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 4));
  int16_t* d_p = ctx->io[0].as<int16_t>(); float* d_a = ctx->io[1].as<float>(); float* d_sa = ctx->io[2].as<float>();
  TD_CUDA(h2d(d_p, p, s, st));
  TD_CUDA(h2d(d_sa, sa, s, st));
  Timer t; t.start(st);
  if (int rc = td_d8flowpathextremeup_deps_dev(ctx, d_p, d_a, s, p_nodata, st)) return rc;
  if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
  if (int rc = td_sweep_begin_dev(ctx, s, st)) return rc;
  if (int rc = td_d8flowpathextremeup_sweep_run_dev(ctx, d_sa, d_a, s, usemax, contcheck, ctx->halo.as<int>(), st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(ssa, d_a, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

// dinfdecayaccum (src/dinfdecayaccum.cpp:61): the D-infinity sweep with the decaying-accumulation algebra.  Single strip.
int td_dinfdecayaccum_host(const float* ang, const float* dm, const float* w, float* dsca, int nx, int ny, float ang_nodata, float dm_nodata,
                           const double* dxc, const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows, int nout) {
  if (int rc = need_device()) return rc;
  if (!ang || !dm || !dsca || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_dinfdecayaccum_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[3].ensure(n * 4));
  float* d_ang = ctx->io[0].as<float>(); float* d_a = ctx->io[1].as<float>(); float* d_dm = ctx->io[3].as<float>(); float* d_w = nullptr;
  const double *d_dx, *d_dy;
  if (int rc = upload_rows(ctx, dxc, dyc, ny, &d_dx, &d_dy, st)) return rc;
  TD_CUDA(h2d(d_ang, ang, s, st));
  TD_CUDA(h2d(d_dm, dm, s, st));
  if (w) { TD_CUDA(ctx->io[2].ensure(n * 4)); d_w = ctx->io[2].as<float>(); TD_CUDA(h2d(d_w, w, s, st)); }
  Timer t; t.start(st);
  if (int rc = td_dinfdecayaccum_deps_dev(ctx, d_ang, d_a, s, ang_nodata, d_dx, d_dy, st)) return rc;
  if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
  if (int rc = td_sweep_begin_dev(ctx, s, st)) return rc;
  if (int rc = td_dinfdecayaccum_sweep_run_dev(ctx, d_ang, d_dm, d_w, d_a, s, dm_nodata, contcheck, d_dx, ctx->halo.as<int>(), st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(dsca, d_a, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

// DinfConcLimAccum (src/DinfConcLimAccum.cpp:61) and DinfTransLimAccum (src/DinfTransLimAccum.cpp:61): the D-infinity sweep with the
// concentration- and transport-limited algebras (7; 8 / 9).  Single strip.
namespace {
// uploads the angles and the row tables into io[0] (the result goes to io[1])
int dinf_sibling_upload(td_ctx* ctx, const td_strip& s, const float* ang, const double* dxc, const double* dyc, const double** d_dx, const double** d_dy,
                        cudaStream_t st) {
  const size_t n = (size_t)Strip(s).cells();
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4));
  if (int rc = upload_rows(ctx, dxc, dyc, s.ny, d_dx, d_dy, st)) return rc;
  TD_CUDA(h2d(ctx->io[0].as<float>(), ang, s, st));
  return TD_OK;
}
}  // namespace
int td_dinfconclimaccum_host(const float* ang, const float* dm, const float* q, const int16_t* dg, float* ctpt, int nx, int ny, float ang_nodata, float dm_nodata,
                             float q_nodata, float csol, const double* dxc, const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows, int nout) {
  if (int rc = need_device()) return rc;
  if (!ang || !dm || !q || !dg || !ctpt || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_dinfconclimaccum_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[2].ensure(n * 4)); TD_CUDA(ctx->io[3].ensure(n * 4)); TD_CUDA(ctx->io[4].ensure(n * 2));
  float* d_q = ctx->io[2].as<float>(); float* d_dm = ctx->io[3].as<float>(); int16_t* d_dg = ctx->io[4].as<int16_t>();
  TD_CUDA(h2d(d_q, q, s, st)); TD_CUDA(h2d(d_dm, dm, s, st)); TD_CUDA(h2d(d_dg, dg, s, st));
  Timer t; t.start(st);
  const double *d_dx, *d_dy;
  if (int rc = dinf_sibling_upload(ctx, s, ang, dxc, dyc, &d_dx, &d_dy, st)) return rc;
  float* d_ang = ctx->io[0].as<float>(); float* d_a = ctx->io[1].as<float>();
  if (int rc = td_dinfconclimaccum_deps_dev(ctx, d_ang, d_a, s, ang_nodata, d_dx, d_dy, st)) return rc;
  if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
  if (int rc = td_sweep_begin_dev(ctx, s, st)) return rc;
  if (int rc = td_dinfconclimaccum_sweep_run_dev(ctx, d_ang, d_dm, d_q, d_dg, d_a, s, dm_nodata, q_nodata, csol, contcheck, d_dx, ctx->halo.as<int>(), st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(ctpt, d_a, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}
int td_dinftranslimaccum_host(const float* ang, const float* tsup, const float* tc, const float* cs, float* tla, float* tdep, float* ctpt, int nx, int ny,
                              float ang_nodata, float tsup_nodata, float tc_nodata, float cs_nodata, const double* dxc, const double* dyc, int contcheck,
                              const int* outlet_cols, const int* outlet_rows, int nout) {
  if (int rc = need_device()) return rc;
  if (!ang || !tsup || !tc || !tla || !tdep || (cs != nullptr) != (ctpt != nullptr) || !dxc || !dyc || nx <= 0 || ny <= 0) {
    td::set_error("td_dinftranslimaccum_host: bad arguments (the concentration input and output come together)");
    return TD_ERR_ARG;
  }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[2].ensure(n * 4)); TD_CUDA(ctx->io[3].ensure(n * 4)); TD_CUDA(ctx->io[4].ensure(n * 4));
  float* d_ts = ctx->io[2].as<float>(); float* d_tc = ctx->io[3].as<float>(); float* d_dep = ctx->io[4].as<float>(); float *d_cs = nullptr, *d_co = nullptr;
  TD_CUDA(h2d(d_ts, tsup, s, st)); TD_CUDA(h2d(d_tc, tc, s, st));
  if (cs) {
    TD_CUDA(ctx->io[5].ensure(n * 4)); TD_CUDA(ctx->io[6].ensure(n * 4));
    d_cs = ctx->io[5].as<float>(); d_co = ctx->io[6].as<float>();
    TD_CUDA(h2d(d_cs, cs, s, st));
  }
  Timer t; t.start(st);
  const double *d_dx, *d_dy;
  if (int rc = dinf_sibling_upload(ctx, s, ang, dxc, dyc, &d_dx, &d_dy, st)) return rc;
  float* d_ang = ctx->io[0].as<float>(); float* d_a = ctx->io[1].as<float>();
  if (int rc = td_dinftranslimaccum_deps_dev(ctx, d_ang, d_a, d_dep, d_co, s, ang_nodata, d_dx, d_dy, st)) return rc;
  if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
  if (int rc = td_sweep_begin_dev(ctx, s, st)) return rc;
  if (int rc = td_dinftranslimaccum_sweep_run_dev(ctx, d_ang, d_ts, d_tc, d_cs, d_a, d_dep, d_co, s, tsup_nodata, tc_nodata, cs_nodata, contcheck, d_dx,
                                                  ctx->halo.as<int>(), st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(tla, d_a, s, st)); TD_CUDA(d2h(tdep, d_dep, s, st));
  if (cs) TD_CUDA(d2h(ctpt, d_co, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

// gridnet (src/gridnet.cpp:55): longest upstream path length, total upstream path length and Strahler order of the D8 flow
// field — three runs of the D8 sweep, one value per cell each (algebras 4, 5, 6).  Single strip.
int td_gridnet_host(const int16_t* p, const int32_t* mask, int thresh, float* plen, float* tlen, int16_t* gord, int nx, int ny, int16_t p_nodata,
                    const double* dxc, const double* dyc, const int* outlet_cols, const int* outlet_rows, int nout) {
  if (int rc = need_device()) return rc;
  if (!p || !plen || !tlen || !gord || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_gridnet_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const Strip ss(s);
  const size_t n = (size_t)ss.cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 2)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[3].ensure(n * 4));
  int16_t* d_p = ctx->io[0].as<int16_t>(); float* d_a = ctx->io[1].as<float>(); float* d_ok = nullptr;
  TD_CUDA(h2d(d_p, p, s, st));
  if (mask) {
    TD_CUDA(ctx->io[2].ensure(n * 4));
    int* d_m = ctx->io[2].as<int>();
    TD_CUDA(h2d(d_m, mask, s, st));
    d_ok = ctx->io[3].as<float>();
    if (int rc = td_gridnet_mask_dev(ctx, d_m, d_ok, s, thresh, st)) return rc;
  }
  std::vector<float> dist((size_t)ny * 8);
  td::gridnet_dist_table(dxc, dyc, ny, dist.data());
  TD_CUDA(ctx->rows.ensure(sizeof(float) * dist.size()));
  float* d_dist = ctx->rows.as<float>();
  TD_CUDA(cudaMemcpyAsync(d_dist, dist.data(), sizeof(float) * dist.size(), cudaMemcpyHostToDevice, st));
  Timer t; t.start(st);
  for (int alg = 4; alg <= 6; ++alg) {
    if (int rc = td_gridnet_deps_dev(ctx, d_p, d_a, s, p_nodata, st)) return rc;
    if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
    if (int rc = td_sweep_begin_dev(ctx, s, st)) return rc;
    if (int rc = td_gridnet_sweep_run_dev(ctx, alg - 4, d_ok, d_dist, d_a, s, nout >= 0, ctx->halo.as<int>(), st)) return rc;
    if (alg == 4) TD_CUDA(d2h(plen, d_a, s, st));
    else if (alg == 5) TD_CUDA(d2h(tlen, d_a, s, st));
    else {
      TD_CUDA(ctx->io[2].ensure(n * 2));
      int16_t* d_g = ctx->io[2].as<int16_t>();
      if (int rc = td_gridnet_order_dev(ctx, d_a, d_p, d_ok, d_g, s, p_nodata, nout >= 0, st)) return rc;
      TD_CUDA(d2h(gord, d_g, s, st));
    }
  }
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

// ---- point-wise consumers (pointwise.cu): device-strip and host-grid level
int td_threshold_dev(td_ctx*, const float* ssa, const float* mask, int16_t* src, td_strip s, float thresh, float ssa_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::launch_threshold(ssa, mask, src, Strip(s), thresh, ssa_nodata, (cudaStream_t)stream);
}
int td_twi_dev(td_ctx* ctx, const float* slp, const float* sca, float* twi, td_strip s, float slp_nodata, float sca_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx) { td::set_error("td_twi_dev: bad arguments"); return TD_ERR_ARG; }
  return td::launch_twi(slp, sca, twi, Strip(s), slp_nodata, sca_nodata, (cudaStream_t)stream, &ctx->pend);
}
int td_slopearea_dev(td_ctx* ctx, const float* slp, const float* sca, float* sa, td_strip s, float m, float n, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx) { td::set_error("td_slopearea_dev: bad arguments"); return TD_ERR_ARG; }
  return td::launch_slopearea(slp, sca, sa, Strip(s), m, n, (cudaStream_t)stream, &ctx->pend);
}
int td_slopearearatio_dev(td_ctx*, const float* slp, const float* sca, float* sar, td_strip s, float sca_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::launch_slopearearatio(slp, sca, sar, Strip(s), sca_nodata, (cudaStream_t)stream);
}
// the two-rasters-in, one-raster-out shape shared by slopearea and slopearearatio (which: 0 = slp^m * sca^n, 1 = slp / sca)
static int two_in_one_out_host(const char* who, int which, const float* slp, const float* sca, float* out, int nx, int ny, float a, float b) {
  if (int rc = need_device()) return rc;
  if (!slp || !sca || !out || nx <= 0 || ny <= 0) { td::set_error(std::string(who) + ": bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 4));
  float* d_slp = ctx->io[0].as<float>(); float* d_sca = ctx->io[1].as<float>(); float* d_out = ctx->io[2].as<float>();
  TD_CUDA(h2d(d_slp, slp, s, st)); TD_CUDA(h2d(d_sca, sca, s, st));
  Timer t; t.start(st);
  if (int rc = which == 0 ? td_slopearea_dev(ctx, d_slp, d_sca, d_out, s, a, b, st) : td_slopearearatio_dev(ctx, d_slp, d_sca, d_out, s, a, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(out, d_out, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}
int td_slopearea_host(const float* slp, const float* sca, float* sa, int nx, int ny, float m, float n) {
  return two_in_one_out_host("td_slopearea_host", 0, slp, sca, sa, nx, ny, m, n);
}
int td_slopearearatio_host(const float* slp, const float* sca, float* sar, int nx, int ny, float sca_nodata) {
  return two_in_one_out_host("td_slopearearatio_host", 1, slp, sca, sar, nx, ny, sca_nodata, 0.f);
}
int td_threshold_host(const float* ssa, const float* mask, int16_t* src, int nx, int ny, float thresh, float ssa_nodata) {
  if (int rc = need_device()) return rc;
  if (!ssa || !src || nx <= 0 || ny <= 0) { td::set_error("td_threshold_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 2));
  float* d_ssa = ctx->io[0].as<float>(); int16_t* d_src = ctx->io[1].as<int16_t>(); float* d_mask = nullptr;
  TD_CUDA(h2d(d_ssa, ssa, s, st));
  if (mask) { TD_CUDA(ctx->io[2].ensure(n * 4)); d_mask = ctx->io[2].as<float>(); TD_CUDA(h2d(d_mask, mask, s, st)); }
  Timer t; t.start(st);
  if (int rc = td_threshold_dev(ctx, d_ssa, d_mask, d_src, s, thresh, ssa_nodata, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(src, d_src, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}
int td_twi_host(const float* slp, const float* sca, float* twi, int nx, int ny, float slp_nodata, float sca_nodata) {
  if (int rc = need_device()) return rc;
  if (!slp || !sca || !twi || nx <= 0 || ny <= 0) { td::set_error("td_twi_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 4));
  float* d_slp = ctx->io[0].as<float>(); float* d_sca = ctx->io[1].as<float>(); float* d_twi = ctx->io[2].as<float>();
  TD_CUDA(h2d(d_slp, slp, s, st)); TD_CUDA(h2d(d_sca, sca, s, st));
  Timer t; t.start(st);
  if (int rc = td_twi_dev(ctx, d_slp, d_sca, d_twi, s, slp_nodata, sca_nodata, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(twi, d_twi, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

// ---- the stream definitions of Peuker-Douglas (peuker.cu) and length-area (pointwise.cu)
int td_peukerdouglas_smooth_dev(td_ctx*, const float* fel, float* sm, td_strip s, float fel_nodata, const float* p, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!fel || !sm || !p) { td::set_error("td_peukerdouglas_smooth_dev: bad arguments"); return TD_ERR_ARG; }
  return td::launch_pd_smooth(fel, sm, Strip(s), fel_nodata, p, (cudaStream_t)stream);
}
int td_peukerdouglas_mark_dev(td_ctx*, const float* sm, int16_t* ss, td_strip s, float fel_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!sm || !ss) { td::set_error("td_peukerdouglas_mark_dev: bad arguments"); return TD_ERR_ARG; }
  return td::launch_pd_mark(sm, ss, Strip(s), fel_nodata, (cudaStream_t)stream);
}
int td_lengtharea_dev(td_ctx* ctx, const float* plen, const int32_t* ad8, int16_t* ss, td_strip s, float m, float y, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !plen || !ad8 || !ss) { td::set_error("td_lengtharea_dev: bad arguments"); return TD_ERR_ARG; }
  return td::launch_lengtharea(plen, ad8, ss, Strip(s), m, y, (cudaStream_t)stream, &ctx->pend);
}
int td_peukerdouglas_host(const float* fel, int16_t* ss, int nx, int ny, float fel_nodata, const float* p) {
  if (int rc = need_device()) return rc;
  if (!fel || !ss || !p || nx <= 0 || ny <= 0) { td::set_error("td_peukerdouglas_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 2));
  float* d_fel = ctx->io[0].as<float>(); float* d_s = ctx->io[1].as<float>(); int16_t* d_ss = ctx->io[2].as<int16_t>();
  TD_CUDA(h2d(d_fel, fel, s, st));
  Timer t; t.start(st);
  if (int rc = td_peukerdouglas_smooth_dev(ctx, d_fel, d_s, s, fel_nodata, p, st)) return rc;
  if (int rc = td_peukerdouglas_mark_dev(ctx, d_s, d_ss, s, fel_nodata, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(ss, d_ss, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}
int td_lengtharea_host(const float* plen, const int32_t* ad8, int16_t* ss, int nx, int ny, float m, float y) {
  if (int rc = need_device()) return rc;
  if (!plen || !ad8 || !ss || nx <= 0 || ny <= 0) { td::set_error("td_lengtharea_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 2));
  float* d_plen = ctx->io[0].as<float>(); int32_t* d_ad8 = ctx->io[1].as<int32_t>(); int16_t* d_ss = ctx->io[2].as<int16_t>();
  TD_CUDA(h2d(d_plen, plen, s, st)); TD_CUDA(h2d(d_ad8, ad8, s, st));
  Timer t; t.start(st);
  if (int rc = td_lengtharea_dev(ctx, d_plen, d_ad8, d_ss, s, m, y, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(ss, d_ss, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

// aread8 + areadinf of one DEM in ONE call with the copies overlapped with the kernels: three streams — host -> device (p, then
// ang), compute (aread8 as soon as p has arrived, areadinf as soon as ang has and aread8 is done), device -> host (ad8 while
// areadinf runs, then sca).  Same kernels, same results as td_aread8_host followed by td_area_host (no weights, no outlets).
// Host rasters should be pinned (cudaHostAlloc / cudaHostRegister) — pageable memory makes the copies synchronous.
int td_contributing_areas_host(const int16_t* p, const float* ang, float* ad8, float* sca, int nx, int ny, int16_t p_nodata, float ang_nodata,
                               const double* dxc, const double* dyc, int contcheck) {
  if (int rc = need_device()) return rc;
  if (!p || !ang || !ad8 || !sca || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_contributing_areas_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  TD_CUDA(ctx->io[0].ensure(n * 2)); TD_CUDA(ctx->io[1].ensure(n * 4)); TD_CUDA(ctx->io[2].ensure(n * 4)); TD_CUDA(ctx->io[3].ensure(n * 4));
  int16_t* d_p = ctx->io[0].as<int16_t>(); float* d_ad8 = ctx->io[1].as<float>(); float* d_ang = ctx->io[2].as<float>(); float* d_sca = ctx->io[3].as<float>();
  struct Streams {
    cudaStream_t in = nullptr, run = nullptr, out = nullptr; cudaEvent_t e[4] = {nullptr, nullptr, nullptr, nullptr}; cudaEvent_t t[12] = {};
    ~Streams() { for (auto& x : e) if (x) cudaEventDestroy(x); for (auto& x : t) if (x) cudaEventDestroy(x); if (in) cudaStreamDestroy(in); if (run) cudaStreamDestroy(run); if (out) cudaStreamDestroy(out); }
  } S;
  TD_CUDA(cudaDeviceSynchronize());          // earlier work of this context (legacy stream) is done before the private streams start
  TD_CUDA(cudaStreamCreateWithFlags(&S.in, cudaStreamNonBlocking)); TD_CUDA(cudaStreamCreateWithFlags(&S.run, cudaStreamNonBlocking));
  TD_CUDA(cudaStreamCreateWithFlags(&S.out, cudaStreamNonBlocking));
  for (auto& x : S.e) TD_CUDA(cudaEventCreateWithFlags(&x, cudaEventDisableTiming));
  const bool trace = getenv("TAUDEM_B200_TRACE") != nullptr;      // timestamps of every copy / tool on its stream
  if (trace) for (auto& x : S.t) TD_CUDA(cudaEventCreate(&x));
  auto mark = [&](int i, cudaStream_t st) { if (trace) cudaEventRecord(S.t[i], st); };
  const double *d_dx, *d_dy;
  if (int rc = upload_rows(ctx, dxc, dyc, ny, &d_dx, &d_dy, S.run)) return rc;
  if (int rc = upload_theta_from_host(ctx, dxc, dyc, ny, ctx->theta, S.run)) return rc;     // every small copy before the rasters travel
  mark(0, S.in);
  TD_CUDA(h2d(d_p, p, s, S.in));     TD_CUDA(cudaEventRecord(S.e[0], S.in)); mark(1, S.in);
  // The HOST waits for p: a stream that waits for an event of the upload stream is only released when that stream's LAST
  // upload is done if more uploads were queued behind the event (measured, TAUDEM_B200_TRACE: aread8 began when ang had
  // arrived) — so nothing is queued behind p until the kernels that need it are running.
  TD_CUDA(cudaEventSynchronize(S.e[0]));
  Timer t; t.start(S.run);
  TD_CUDA(cudaStreamWaitEvent(S.run, S.e[0], 0));
  mark(3, S.run);
  if (int rc = td_aread8_deps_dev(ctx, d_p, d_ad8, s, p_nodata, S.run)) return rc;
  if (int rc = td_aread8_sweep_dev(ctx, nullptr, d_ad8, s, 0.f, 0, contcheck, S.run)) return rc;
  TD_CUDA(cudaEventRecord(S.e[2], S.run)); mark(4, S.run);
  (void)cudaStreamQuery(S.run);                      // push the launches to the device now
  const auto h0 = std::chrono::steady_clock::now();
  TD_CUDA(h2d(d_ang, ang, s, S.in)); TD_CUDA(cudaEventRecord(S.e[1], S.in)); mark(2, S.in);
  if (trace) fprintf(stderr, "[td trace] host spent %.2f ms enqueueing the ang upload\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count());
  TD_CUDA(cudaStreamWaitEvent(S.out, S.e[2], 0));
  mark(5, S.out);
  TD_CUDA(d2h(ad8, d_ad8, s, S.out));
  mark(6, S.out);
  TD_CUDA(cudaStreamWaitEvent(S.run, S.e[1], 0));
  mark(7, S.run);
  if (int rc = area_deps(ctx, d_ang, d_sca, s, ang_nodata, d_dx, d_dy, true, S.run)) return rc;
  if (int rc = td_area_sweep_dev(ctx, d_ang, nullptr, d_sca, s, 0, contcheck, d_dx, S.run)) return rc;
  TD_CUDA(cudaEventRecord(S.e[3], S.run)); mark(8, S.run);
  td::set_compute_seconds(t.stop(S.run));
  TD_CUDA(cudaStreamWaitEvent(S.out, S.e[3], 0));
  mark(9, S.out);
  TD_CUDA(d2h(sca, d_sca, s, S.out));
  mark(10, S.out);
  TD_CUDA(cudaStreamSynchronize(S.out));
  TD_CUDA(cudaStreamSynchronize(S.in));
  if (trace) {
    const char* what[11] = {"in: start", "in: p arrived", "in: ang arrived", "run: aread8 starts", "run: aread8 done", "out: ad8 copy starts", "out: ad8 copied",
                            "run: areadinf starts", "run: areadinf done", "out: sca copy starts", "out: sca copied"};
    for (int i = 1; i < 11; ++i) { float ms = 0; cudaEventElapsedTime(&ms, S.t[0], S.t[i]); fprintf(stderr, "[td trace] %8.2f ms  %s\n", ms, what[i]); }
  }
  return TD_OK;
}

int td_area_host(const float* ang, const float* w, float* sca, int nx, int ny, float ang_nodata, float w_nodata, const double* dxc,
                 const double* dyc, int contcheck) {
  return td_area_outlets_host(ang, w, sca, nx, ny, ang_nodata, w_nodata, dxc, dyc, contcheck, nullptr, nullptr, -1);
}

int td_area_outlets_host(const float* ang, const float* w, float* sca, int nx, int ny, float ang_nodata, float w_nodata, const double* dxc,
                         const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows, int nout) {
  (void)w_nodata;   // the reference adds the raw weight, nodata or not (src/areadinf.cpp:210)
  if (int rc = need_device()) return rc;
  if (!ang || !sca || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_area_host: bad arguments"); return TD_ERR_ARG; }
  td_ctx* ctx = default_ctx();
  const td_strip s = host_strip(nx, ny);
  const size_t n = (size_t)Strip(s).cells();
  cudaStream_t st = 0;
  TD_CUDA(ctx->io[0].ensure(n * 4)); TD_CUDA(ctx->io[1].ensure(n * 4));
  float* d_ang = ctx->io[0].as<float>(); float* d_a = ctx->io[1].as<float>(); float* d_w = nullptr;
  const double *d_dx, *d_dy;
  if (int rc = upload_rows(ctx, dxc, dyc, ny, &d_dx, &d_dy, st)) return rc;
  TD_CUDA(h2d(d_ang, ang, s, st));
  if (w) { TD_CUDA(ctx->io[2].ensure(n * 4)); d_w = ctx->io[2].as<float>(); TD_CUDA(h2d(d_w, w, s, st)); }
  Timer t; t.start(st);
  if (int rc = td_area_deps_dev(ctx, d_ang, d_a, s, ang_nodata, d_dx, d_dy, st)) return rc;
  if (nout >= 0) { if (int rc = td_sweep_restrict_dev(ctx, s, outlet_cols, outlet_rows, nout, st)) return rc; }
  if (int rc = td_area_sweep_dev(ctx, d_ang, d_w, d_a, s, w != nullptr, contcheck, d_dx, st)) return rc;
  td::set_compute_seconds(t.stop(st));
  TD_CUDA(d2h(sca, d_a, s, st));
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}

}  // extern "C"
