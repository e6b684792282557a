// C ABI of taudem_b200: device-strip level and host-grid level entry points
// (declared in include/taudem_b200.h).  File-level entry points live in tools.cpp.
#include <math.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <iterator>
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
// flowdircond: the aread8 dependency state of p (the reference's queue is initNeighborD8up's, src/flowdircond.cpp:138), the output
// starting as a copy of z (src/flowdircond.cpp:154-172 lowers z in place; cells the queue never reaches keep their z)
int td_flowdircond_deps_dev(td_ctx* ctx, const int16_t* p, const float* z, float* zfdc, td_strip s, int16_t p_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!p || !z || !zfdc) { td::set_error("td_flowdircond_deps_dev: bad arguments"); return TD_ERR_ARG; }
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = ensure_dep_state(ctx, Strip(s), st)) return rc;
  ctx->sweep_dinf = 0;
  TD_CUDA(td::launch_deps_d8(p, ctx->node.as<unsigned short>(), ctx->cnt.as<unsigned char>(), zfdc, Strip(s), p_nodata, st));
  TD_CUDA(cudaMemcpyAsync(zfdc, z, sizeof(float) * (size_t)Strip(s).cells(), cudaMemcpyDeviceToDevice, st));
  return TD_OK;
}
int td_flowdircond_sweep_run_dev(td_ctx* ctx, const float* z, float* zfdc, td_strip s, float z_nodata, int* halo_out, void* stream) {
  if (int rc = check_strip(s)) return rc;
  return td::wsweep_run(ctx, false, zfdc, z, nullptr, Strip(s), z_nodata, 1, 0, nullptr, nullptr, halo_out, (cudaStream_t)stream, 11);
}
// retlimflow's gather reads a contributor's share with prop() without testing its angle for nodata (src/RetlimFlow.cpp:155-163):
// a nodata value that prop() reads as a direction would add p * MISSINGFLOAT.  Such a value is refused, decided with prop() itself
// (src/commonLib.cpp:76-91) on the cell sizes of every row a contributor can lie in (the strip's rows and its neighbours' edge rows).
static double prop_host(float a, int k, double dx1, double dy1) {
  double aref[10] = {-atan2(dy1, dx1), 0., 0., 0.5 * TD_PI, 0., TD_PI, 0., 1.5 * TD_PI, 0., 2. * TD_PI};
  aref[2] = -aref[0]; aref[4] = TD_PI - aref[2]; aref[6] = TD_PI + aref[2]; aref[8] = 2. * TD_PI - aref[2];
  double p = 0.;
  if (k == 1 && a > TD_PI) a = (float)(a - 2.0 * TD_PI);
  if (a > aref[k - 1] && a < aref[k + 1]) p = a > aref[k] ? (aref[k + 1] - a) / (aref[k + 1] - aref[k]) : (a - aref[k - 1]) / (aref[k] - aref[k - 1]);
  return p < 1e-5 ? -1. : p;
}
static int check_ang_nodata(td_ctx* ctx, const td_strip& s, float ang_nodata, const double* dxc, const double* dyc) {
  std::vector<double> dx((size_t)s.ny + 2), dy((size_t)s.ny + 2);
  TD_CUDA(cudaMemcpy(dx.data(), dxc, sizeof(double) * s.ny, cudaMemcpyDeviceToHost));
  TD_CUDA(cudaMemcpy(dy.data(), dyc, sizeof(double) * s.ny, cudaMemcpyDeviceToHost));
  int n = s.ny;
  for (int i = 0; i < 2; ++i)
    if (ctx->halo_dx[i] > 0. && ctx->halo_dy[i] > 0.) { dx[n] = ctx->halo_dx[i]; dy[n] = ctx->halo_dy[i]; ++n; }
  for (int r = 0; r < n; ++r) {
    if (r > 0 && dx[r] == dx[r - 1] && dy[r] == dy[r - 1]) continue;
    for (int k = 1; k <= 8; ++k)
      if (prop_host(ang_nodata, k, dx[r], dy[r]) > 0.) {
        td::set_error("retlimflow: the angle nodata value " + std::to_string(ang_nodata) + " is a flow direction to prop(); the reference would add its "
                      "share times MISSINGFLOAT (use a nodata value below -pi/4, e.g. -FLT_MAX)");
        return TD_ERR_ARG;
      }
  }
  return TD_OK;
}
// retlimflow: the areadinf dependency state of ang (initNeighborDinfup, src/RetlimFlow.cpp:128), qrl starting as MISSINGFLOAT,
// then the cells whose wg or rc is nodata blocked (launch_block_cells)
int td_retlimflow_deps_dev(td_ctx* ctx, const float* ang, const float* wg, const float* rc, float* qrl, td_strip s, float ang_nodata, float wg_nodata,
                           float rc_nodata, const double* dxc, const double* dyc, void* stream) {
  if (int rc_ = check_strip(s)) return rc_;
  if (!ang || !wg || !rc || !qrl || !dxc || !dyc) { td::set_error("td_retlimflow_deps_dev: bad arguments"); return TD_ERR_ARG; }
  if (int e = check_ang_nodata(ctx, s, ang_nodata, dxc, dyc)) return e;
  if (int e = area_deps(ctx, ang, qrl, s, ang_nodata, dxc, dyc, false, stream, TD_MISSINGFLOAT)) return e;
  TD_CUDA(td::launch_block_cells(ctx->node.as<unsigned short>(), wg, wg_nodata, rc, rc_nodata, Strip(s), (cudaStream_t)stream));
  return TD_OK;
}
int td_retlimflow_sweep_run_dev(td_ctx* ctx, const float* ang, const float* wg, const float* rc, float* qrl, td_strip s, float wg_nodata, float rc_nodata,
                                const double* dxc, int* halo_out, void* stream) {
  if (int e = check_strip(s)) return e;
  return td::wsweep_run(ctx, true, qrl, wg, ang, Strip(s), wg_nodata, 1, 0, ctx->theta.as<double>(), dxc, halo_out, (cudaStream_t)stream, 12, rc,
                        rc_nodata);
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

// A failed step of a host-grid call, with its return code (the message is recorded already).  Thrown, so that nothing runs after it.
struct Stop { int rc; };
#define HG_CUDA(call)                                                             \
  do {                                                                            \
    const cudaError_t e__ = (call);                                               \
    if (e__ != cudaSuccess) throw Stop{::td::cuda_fail(e__, #call)};              \
  } while (0)
#define HG_TD(call)                                                               \
  do {                                                                            \
    if (const int rc__ = (call)) throw Stop{rc__};                                \
  } while (0)

// One host-grid call on the default context and the legacy stream.  Every raster of the call gets the next of the context's io slots,
// so no two live rasters share one; the device compute time runs from start() (after the uploads) to stop() (before the downloads).
struct HostGrid {
  td_ctx* ctx = default_ctx();
  td_strip s;
  cudaStream_t st = 0;
  Timer timer;
  size_t slot = 0;
  HostGrid(int nx, int ny) : s(host_strip(nx, ny)) {}

  // a strip of per_cell T's per cell
  template <typename T> T* alloc(size_t per_cell = 1) {
    if (slot == std::size(ctx->io)) { td::set_error("host-grid call: more rasters than io slots"); throw Stop{TD_ERR_ARG}; }
    td_ctx::Buf& b = ctx->io[slot++];
    HG_CUDA(b.ensure(sizeof(T) * per_cell * (size_t)Strip(s).cells()));
    return b.as<T>();
  }
  template <typename T> void up(T* d, const T* h) { HG_CUDA(h2d(d, h, s, st)); }
  template <typename T> void down(T* h, const T* d) { HG_CUDA(d2h(h, d, s, st)); }
  // an input raster on the device; an optional input that is not given (NULL) takes no slot
  template <typename T> T* in(const T* h) {
    if (!h) return nullptr;
    T* d = alloc<T>();
    up(d, h);
    return d;
  }
  void cell_sizes(const double* dxc, const double* dyc, const double** d_dx, const double** d_dy) {
    HG_TD(upload_rows(ctx, dxc, dyc, s.ny, d_dx, d_dy, st));
  }
  // the cell-to-cell distances of every row (td::gridnet_dist_table) that gridnet and slopeavedown read
  const float* dist(const double* dxc, const double* dyc) {
    std::vector<float> d((size_t)s.ny * 8);
    td::gridnet_dist_table(dxc, dyc, s.ny, d.data());
    HG_CUDA(ctx->rows.ensure(sizeof(float) * d.size()));
    HG_CUDA(cudaMemcpyAsync(ctx->rows.p, d.data(), sizeof(float) * d.size(), cudaMemcpyHostToDevice, st));
    return ctx->rows.as<float>();
  }
  void start() { timer.start(st); }
  void stop() { td::set_compute_seconds(timer.stop(st)); }
  // -o: between a sweep's deps and its run, only the cells upstream of the outlets (nout >= 0)
  void restrict_to(const int* cols, const int* rows, int nout) {
    if (nout >= 0) HG_TD(td_sweep_restrict_dev(ctx, s, cols, rows, nout, st));
  }
  // the same, then every tile queued: what follows a deps call before a *_sweep_run_dev into halo()
  void begin_sweep(const int* cols = nullptr, const int* rows = nullptr, int nout = -1) {
    restrict_to(cols, rows, nout);
    HG_TD(td_sweep_begin_dev(ctx, s, st));
  }
  int* halo() const { return ctx->halo.as<int>(); }
};

// the device check, then the argument check (args_ok and the grid's size), then body(g); ends with the legacy stream synchronized
template <class Body>
int host_call(const char* who, bool args_ok, int nx, int ny, Body&& body, const char* arg_hint = "") {
  if (int rc = need_device()) return rc;
  if (!args_ok || nx <= 0 || ny <= 0) { td::set_error(std::string(who) + ": bad arguments" + arg_hint); return TD_ERR_ARG; }
  try {
    HostGrid g(nx, ny);
    body(g);
    HG_CUDA(cudaStreamSynchronize(g.st));
  } catch (const Stop& e) {
    return e.rc;
  }
  return TD_OK;
}
}  // namespace

extern "C" {

int td_flood_host(const float* dem, float* fel, const int16_t* depmask, int nx, int ny, float dem_nodata, int is_4Point) {
  return host_call("td_flood_host", dem && fel, nx, ny, [&](HostGrid& g) {
    const float* d_dem = g.in(dem);
    float* d_fel = g.alloc<float>();
    const int16_t* d_mask = g.in(depmask);
    g.start();
    HG_TD(td_flood_init_dev(g.ctx, d_dem, d_mask, d_fel, g.s, dem_nodata, is_4Point, g.st));
    int changed = 0;
    HG_TD(td_flood_relax_dev(g.ctx, d_dem, d_fel, g.s, is_4Point, &changed, g.st));
    g.stop();
    g.down(fel, d_fel);
  });
}

int td_setdird8_host(const float* fel, int16_t* p, float* sd8, int nx, int ny, float fel_nodata, const double* dxc, const double* dyc) {
  return host_call("td_setdird8_host", fel && p && sd8 && dxc && dyc, nx, ny, [&](HostGrid& g) {
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    float* d_fel = g.in(fel);
    float* d_sd8 = g.alloc<float>();
    int16_t* d_p = g.alloc<int16_t>();
    g.start();
    long long nflat = 0;
    HG_TD(td_d8_slopes_dev(g.ctx, d_fel, d_p, d_sd8, g.s, fel_nodata, d_dx, d_dy, &nflat, g.st));
    // the slope raster is final before flats are resolved (src/d8.cpp:282-288)
    if (nflat > 0) { long long left = 0; HG_TD(td_d8_flats_dev(g.ctx, d_fel, d_p, g.s, d_dx, d_dy, &left, g.st)); }
    g.stop();
    g.down(p, d_p);
    g.down(sd8, d_sd8);
  });
}

int td_setdir_host(const float* fel, float* ang, float* slp, int nx, int ny, float fel_nodata, const double* dxc, const double* dyc) {
  return host_call("td_setdir_host", fel && ang && slp && dxc && dyc, nx, ny, [&](HostGrid& g) {
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    float* d_fel = g.in(fel);
    float* d_slp = g.alloc<float>();
    float* d_ang = g.alloc<float>();
    g.start();
    long long nflat = 0;
    HG_TD(td_dinf_slopes_dev(g.ctx, d_fel, d_ang, d_slp, g.s, fel_nodata, d_dx, d_dy, &nflat, g.st));
    if (nflat > 0) { long long left = 0; HG_TD(td_dinf_flats_dev(g.ctx, d_fel, d_ang, g.s, d_dx, d_dy, &left, g.st)); }
    g.stop();
    g.down(ang, d_ang);
    g.down(slp, d_slp);
  });
}

int td_aread8_host(const int16_t* p, const float* w, float* ad8, int nx, int ny, int16_t p_nodata, float w_nodata, int contcheck) {
  return td_aread8_outlets_host(p, w, ad8, nx, ny, p_nodata, w_nodata, contcheck, nullptr, nullptr, -1);
}

// nout < 0: no outlets (the whole grid); nout >= 0: only the cells upstream of the outlets (src/aread8.cpp -o)
int td_aread8_outlets_host(const int16_t* p, const float* w, float* ad8, int nx, int ny, int16_t p_nodata, float w_nodata, int contcheck,
                           const int* outlet_cols, const int* outlet_rows, int nout) {
  trace_mark("aread8_host: enter");
  const int rc = host_call("td_aread8_host", p && ad8, nx, ny, [&](HostGrid& g) {
    trace_mark("aread8_host: device ready");
    int16_t* d_p = g.alloc<int16_t>();
    float* d_ad8 = g.alloc<float>();
    trace_mark("aread8_host: buffers allocated");
    g.up(d_p, p);
    const float* d_w = g.in(w);
    if (getenv("TAUDEM_B200_TRACE")) { cudaStreamSynchronize(g.st); trace_mark("aread8_host: inputs on the device"); }
    g.start();
    HG_TD(td_aread8_deps_dev(g.ctx, d_p, d_ad8, g.s, p_nodata, g.st));
    g.restrict_to(outlet_cols, outlet_rows, nout);
    HG_TD(td_aread8_sweep_dev(g.ctx, d_w, d_ad8, g.s, w_nodata, w != nullptr, contcheck, g.st));
    g.stop();
    trace_mark("aread8_host: computed");
    g.down(ad8, d_ad8);
  });
  if (rc == TD_OK) trace_mark("aread8_host: result on the host");
  return rc;
}

// ---- d8flowpathextremeup (src/D8flowpathextremeup.cpp:58-285): the D8 dependency stencil and sweep with the extreme-value
// algebra — each cell gets the largest (usemax) / smallest value of `sa` on the flow paths that end in it; nodata = MISSINGFLOAT.
int td_d8flowpathextremeup_host(const int16_t* p, const float* sa, float* ssa, int nx, int ny, int16_t p_nodata, int usemax, int contcheck,
                                const int* outlet_cols, const int* outlet_rows, int nout) {
  return host_call("td_d8flowpathextremeup_host", p && sa && ssa, nx, ny, [&](HostGrid& g) {
    const int16_t* d_p = g.in(p);
    const float* d_sa = g.in(sa);
    float* d_ssa = g.alloc<float>();
    g.start();
    HG_TD(td_d8flowpathextremeup_deps_dev(g.ctx, d_p, d_ssa, g.s, p_nodata, g.st));
    g.begin_sweep(outlet_cols, outlet_rows, nout);
    HG_TD(td_d8flowpathextremeup_sweep_run_dev(g.ctx, d_sa, d_ssa, g.s, usemax, contcheck, g.halo(), g.st));
    g.stop();
    g.down(ssa, d_ssa);
  });
}

// ---- flowdircond (src/flowdircond.cpp:56-194): the D8 dependency stencil and sweep of p with the conditioning algebra (11).
int td_flowdircond_host(const int16_t* p, const float* z, float* zfdc, int nx, int ny, int16_t p_nodata, float z_nodata) {
  return host_call("td_flowdircond_host", p && z && zfdc, nx, ny, [&](HostGrid& g) {
    const int16_t* d_p = g.in(p);
    const float* d_z = g.in(z);
    float* d_zfdc = g.alloc<float>();
    g.start();
    HG_TD(td_flowdircond_deps_dev(g.ctx, d_p, d_z, d_zfdc, g.s, p_nodata, g.st));
    g.begin_sweep();
    HG_TD(td_flowdircond_sweep_run_dev(g.ctx, d_z, d_zfdc, g.s, z_nodata, g.halo(), g.st));
    g.stop();
    g.down(zfdc, d_zfdc);
  });
}

// ---- retlimflow (src/RetlimFlow.cpp:53-240): the D-infinity dependency stencil and sweep with the retention-limited algebra (12).
int td_retlimflow_host(const float* ang, const float* wg, const float* rc, float* qrl, int nx, int ny, float ang_nodata, float wg_nodata, float rc_nodata,
                       const double* dxc, const double* dyc) {
  return host_call("td_retlimflow_host", ang && wg && rc && qrl && dxc && dyc, nx, ny, [&](HostGrid& g) {
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    const float* d_ang = g.in(ang);
    const float* d_wg = g.in(wg);
    const float* d_rc = g.in(rc);
    float* d_qrl = g.alloc<float>();
    g.start();
    HG_TD(td_retlimflow_deps_dev(g.ctx, d_ang, d_wg, d_rc, d_qrl, g.s, ang_nodata, wg_nodata, rc_nodata, d_dx, d_dy, g.st));
    g.begin_sweep();
    HG_TD(td_retlimflow_sweep_run_dev(g.ctx, d_ang, d_wg, d_rc, d_qrl, g.s, wg_nodata, rc_nodata, d_dx, g.halo(), g.st));
    g.stop();
    g.down(qrl, d_qrl);
  });
}

// dinfdecayaccum (src/dinfdecayaccum.cpp:61): the D-infinity sweep with the decaying-accumulation algebra.  Single strip.
int td_dinfdecayaccum_host(const float* ang, const float* dm, const float* w, float* dsca, int nx, int ny, float ang_nodata, float dm_nodata,
                           const double* dxc, const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows, int nout) {
  return host_call("td_dinfdecayaccum_host", ang && dm && dsca && dxc && dyc, nx, ny, [&](HostGrid& g) {
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    const float* d_ang = g.in(ang);
    const float* d_dm = g.in(dm);
    const float* d_w = g.in(w);
    float* d_dsca = g.alloc<float>();
    g.start();
    HG_TD(td_dinfdecayaccum_deps_dev(g.ctx, d_ang, d_dsca, g.s, ang_nodata, d_dx, d_dy, g.st));
    g.begin_sweep(outlet_cols, outlet_rows, nout);
    HG_TD(td_dinfdecayaccum_sweep_run_dev(g.ctx, d_ang, d_dm, d_w, d_dsca, g.s, dm_nodata, contcheck, d_dx, g.halo(), g.st));
    g.stop();
    g.down(dsca, d_dsca);
  });
}

// DinfConcLimAccum (src/DinfConcLimAccum.cpp:61) and DinfTransLimAccum (src/DinfTransLimAccum.cpp:61): the D-infinity sweep with the
// concentration- and transport-limited algebras (7; 8 / 9).  Single strip.
int td_dinfconclimaccum_host(const float* ang, const float* dm, const float* q, const int16_t* dg, float* ctpt, int nx, int ny, float ang_nodata, float dm_nodata,
                             float q_nodata, float csol, const double* dxc, const double* dyc, int contcheck, const int* outlet_cols, const int* outlet_rows, int nout) {
  return host_call("td_dinfconclimaccum_host", ang && dm && q && dg && ctpt && dxc && dyc, nx, ny, [&](HostGrid& g) {
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    const float* d_ang = g.in(ang);
    const float* d_dm = g.in(dm);
    const float* d_q = g.in(q);
    const int16_t* d_dg = g.in(dg);
    float* d_ctpt = g.alloc<float>();
    g.start();
    HG_TD(td_dinfconclimaccum_deps_dev(g.ctx, d_ang, d_ctpt, g.s, ang_nodata, d_dx, d_dy, g.st));
    g.begin_sweep(outlet_cols, outlet_rows, nout);
    HG_TD(td_dinfconclimaccum_sweep_run_dev(g.ctx, d_ang, d_dm, d_q, d_dg, d_ctpt, g.s, dm_nodata, q_nodata, csol, contcheck, d_dx, g.halo(), g.st));
    g.stop();
    g.down(ctpt, d_ctpt);
  });
}
int td_dinftranslimaccum_host(const float* ang, const float* tsup, const float* tc, const float* cs, float* tla, float* tdep, float* ctpt, int nx, int ny,
                              float ang_nodata, float tsup_nodata, float tc_nodata, float cs_nodata, const double* dxc, const double* dyc, int contcheck,
                              const int* outlet_cols, const int* outlet_rows, int nout) {
  const bool args_ok = ang && tsup && tc && tla && tdep && (cs != nullptr) == (ctpt != nullptr) && dxc && dyc;
  return host_call("td_dinftranslimaccum_host", args_ok, nx, ny, [&](HostGrid& g) {
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    const float* d_ang = g.in(ang);
    const float* d_tsup = g.in(tsup);
    const float* d_tc = g.in(tc);
    const float* d_cs = g.in(cs);
    float* d_tla = g.alloc<float>();
    float* d_tdep = g.alloc<float>();
    float* d_ctpt = cs ? g.alloc<float>() : nullptr;
    g.start();
    HG_TD(td_dinftranslimaccum_deps_dev(g.ctx, d_ang, d_tla, d_tdep, d_ctpt, g.s, ang_nodata, d_dx, d_dy, g.st));
    g.begin_sweep(outlet_cols, outlet_rows, nout);
    HG_TD(td_dinftranslimaccum_sweep_run_dev(g.ctx, d_ang, d_tsup, d_tc, d_cs, d_tla, d_tdep, d_ctpt, g.s, tsup_nodata, tc_nodata, cs_nodata, contcheck, d_dx,
                                             g.halo(), g.st));
    g.stop();
    g.down(tla, d_tla);
    g.down(tdep, d_tdep);
    if (cs) g.down(ctpt, d_ctpt);
  }, " (the concentration input and output come together)");
}

// gridnet (src/gridnet.cpp:55): longest upstream path length, total upstream path length and Strahler order of the D8 flow
// field — three runs of the D8 sweep, one value per cell each (algebras 4, 5, 6).  Single strip.  The three sweeps share one
// buffer, so each result is downloaded as soon as it is complete (inside the timed region).
int td_gridnet_host(const int16_t* p, const int32_t* mask, int thresh, float* plen, float* tlen, int16_t* gord, int nx, int ny, int16_t p_nodata,
                    const double* dxc, const double* dyc, const int* outlet_cols, const int* outlet_rows, int nout) {
  return host_call("td_gridnet_host", p && plen && tlen && gord && dxc && dyc, nx, ny, [&](HostGrid& g) {
    const int16_t* d_p = g.in(p);
    float* d_len = g.alloc<float>();
    float* d_ok = nullptr;
    if (mask) {
      const int32_t* d_mask = g.in(mask);
      d_ok = g.alloc<float>();
      HG_TD(td_gridnet_mask_dev(g.ctx, d_mask, d_ok, g.s, thresh, g.st));
    }
    const float* d_dist = g.dist(dxc, dyc);
    int16_t* d_gord = g.alloc<int16_t>();
    g.start();
    for (int which = 0; which < 3; ++which) {
      HG_TD(td_gridnet_deps_dev(g.ctx, d_p, d_len, g.s, p_nodata, g.st));
      g.begin_sweep(outlet_cols, outlet_rows, nout);
      HG_TD(td_gridnet_sweep_run_dev(g.ctx, which, d_ok, d_dist, d_len, g.s, nout >= 0, g.halo(), g.st));
      if (which < 2) g.down(which == 0 ? plen : tlen, d_len);
    }
    HG_TD(td_gridnet_order_dev(g.ctx, d_len, d_p, d_ok, d_gord, g.s, p_nodata, nout >= 0, g.st));
    g.down(gord, d_gord);
    g.stop();
  });
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
int td_slopearea_host(const float* slp, const float* sca, float* sa, int nx, int ny, float m, float n) {
  return host_call("td_slopearea_host", slp && sca && sa, nx, ny, [&](HostGrid& g) {
    const float* d_slp = g.in(slp);
    const float* d_sca = g.in(sca);
    float* d_sa = g.alloc<float>();
    g.start();
    HG_TD(td_slopearea_dev(g.ctx, d_slp, d_sca, d_sa, g.s, m, n, g.st));
    g.stop();
    g.down(sa, d_sa);
  });
}
int td_slopearearatio_host(const float* slp, const float* sca, float* sar, int nx, int ny, float sca_nodata) {
  return host_call("td_slopearearatio_host", slp && sca && sar, nx, ny, [&](HostGrid& g) {
    const float* d_slp = g.in(slp);
    const float* d_sca = g.in(sca);
    float* d_sar = g.alloc<float>();
    g.start();
    HG_TD(td_slopearearatio_dev(g.ctx, d_slp, d_sca, d_sar, g.s, sca_nodata, g.st));
    g.stop();
    g.down(sar, d_sar);
  });
}
int td_threshold_host(const float* ssa, const float* mask, int16_t* src, int nx, int ny, float thresh, float ssa_nodata) {
  return host_call("td_threshold_host", ssa && src, nx, ny, [&](HostGrid& g) {
    const float* d_ssa = g.in(ssa);
    int16_t* d_src = g.alloc<int16_t>();
    const float* d_mask = g.in(mask);
    g.start();
    HG_TD(td_threshold_dev(g.ctx, d_ssa, d_mask, d_src, g.s, thresh, ssa_nodata, g.st));
    g.stop();
    g.down(src, d_src);
  });
}
int td_twi_host(const float* slp, const float* sca, float* twi, int nx, int ny, float slp_nodata, float sca_nodata) {
  return host_call("td_twi_host", slp && sca && twi, nx, ny, [&](HostGrid& g) {
    const float* d_slp = g.in(slp);
    const float* d_sca = g.in(sca);
    float* d_twi = g.alloc<float>();
    g.start();
    HG_TD(td_twi_dev(g.ctx, d_slp, d_sca, d_twi, g.s, slp_nodata, sca_nodata, g.st));
    g.stop();
    g.down(twi, d_twi);
  });
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
  return host_call("td_peukerdouglas_host", fel && ss && p, nx, ny, [&](HostGrid& g) {
    const float* d_fel = g.in(fel);
    float* d_sm = g.alloc<float>();
    int16_t* d_ss = g.alloc<int16_t>();
    g.start();
    HG_TD(td_peukerdouglas_smooth_dev(g.ctx, d_fel, d_sm, g.s, fel_nodata, p, g.st));
    HG_TD(td_peukerdouglas_mark_dev(g.ctx, d_sm, d_ss, g.s, fel_nodata, g.st));
    g.stop();
    g.down(ss, d_ss);
  });
}
int td_lengtharea_host(const float* plen, const int32_t* ad8, int16_t* ss, int nx, int ny, float m, float y) {
  return host_call("td_lengtharea_host", plen && ad8 && ss, nx, ny, [&](HostGrid& g) {
    const float* d_plen = g.in(plen);
    const int32_t* d_ad8 = g.in(ad8);
    int16_t* d_ss = g.alloc<int16_t>();
    g.start();
    HG_TD(td_lengtharea_dev(g.ctx, d_plen, d_ad8, d_ss, g.s, m, y, g.st));
    g.stop();
    g.down(ss, d_ss);
  });
}

// ---- slopeavedown (slopeavedown.cu): the D8 sweep marks the cells the reference's queue processes, then the passes
// niter = (int)(dn / min(dx, dy) + 1) (src/SlopeAveDown.cpp:172); TD_ERR_ARG where the reference's conversion is undefined
int td_slopeavedown_niter(double dn, double dx, double dy, int* niter) {
  const double v = dn / std::min(dx, dy) + 1;
  if (!niter || !isfinite(dn) || !(v > -2147483649.0 && v < 2147483648.0)) {
    td::set_error("slopeavedown: dn / min(dx, dy) + 1 is not a finite number that fits an int");
    return TD_ERR_ARG;
  }
  *niter = (int)v;
  return TD_OK;
}
int td_slopeavedown_init_dev(td_ctx* ctx, const int16_t* p, const float* fel, uint8_t* code, float* ed_dd0, float* ed_dd1, float* sd, td_strip s,
                             int16_t p_nodata, float fel_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !p || !fel || !code || !ed_dd0 || !ed_dd1 || !sd || ed_dd0 == ed_dd1 || !ctx->cnt.p || ctx->sweep_dinf) {
    td::set_error("td_slopeavedown_init_dev: bad arguments (the D8 dependency stencil and sweep of p come first, on this context)");
    return TD_ERR_ARG;
  }
  return td::launch_sad_init(p, ctx->cnt.as<unsigned char>(), fel, code, ed_dd0, ed_dd1, sd, Strip(s), p_nodata, fel_nodata, (cudaStream_t)stream);
}
int td_slopeavedown_pass_dev(td_ctx* ctx, const uint8_t* code, const float* fel, const float* ed_dd_in, float* ed_dd_out, float* sd, td_strip s,
                             const float* dist, double dn, int* changed, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !code || !fel || !ed_dd_in || !ed_dd_out || !sd || !dist || ed_dd_in == ed_dd_out) {
    td::set_error("td_slopeavedown_pass_dev: bad arguments");
    return TD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int* d_flag = reinterpret_cast<int*>(ctx->d_ctr + 36);
  TD_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), st));
  if (int rc = td::launch_sad_pass(code, fel, ed_dd_in, ed_dd_out, sd, dist, Strip(s), dn, d_flag, st)) return rc;
  if (changed) {
    TD_CUDA(cudaMemcpyAsync(ctx->h_ctr + 36, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    TD_CUDA(cudaStreamSynchronize(st));
    *changed = *reinterpret_cast<const int*>(ctx->h_ctr + 36) != 0;
  }
  return TD_OK;
}
// src/SlopeAveDown.cpp:59-330 on one strip: the D8 sweep, then at most niter passes (none after the first that changes nothing)
int td_slopeavedown_host(const float* fel, const int16_t* p, float* slpd, int nx, int ny, float fel_nodata, int16_t p_nodata, const double* dxc,
                         const double* dyc, double dx, double dy, double dn) {
  return host_call("td_slopeavedown_host", fel && p && slpd && dxc && dyc, nx, ny, [&](HostGrid& g) {
    int niter = 0;
    HG_TD(td_slopeavedown_niter(dn, dx, dy, &niter));
    const float* d_dist = g.dist(dxc, dyc);
    const int16_t* d_p = g.in(p);
    const float* d_fel = g.in(fel);
    float* d_sd = g.alloc<float>();                    // the sweep's area scratch first, then the slopes
    uint8_t* d_code = g.alloc<uint8_t>();
    float* d_state[2] = {g.alloc<float>(2), g.alloc<float>(2)};
    g.start();
    HG_TD(td_aread8_deps_dev(g.ctx, d_p, d_sd, g.s, p_nodata, g.st));
    HG_TD(td_aread8_sweep_dev(g.ctx, nullptr, d_sd, g.s, 0.f, 0, 0, g.st));
    HG_TD(td_slopeavedown_init_dev(g.ctx, d_p, d_fel, d_code, d_state[0], d_state[1], d_sd, g.s, p_nodata, fel_nodata, g.st));
    for (int it = 0; it < niter; ++it) {
      int changed = 0;
      HG_TD(td_slopeavedown_pass_dev(g.ctx, d_code, d_fel, d_state[it & 1], d_state[(it + 1) & 1], d_sd, g.s, d_dist, dn, &changed, g.st));
      if (!changed) break;                             // a fixed point: the remaining passes would change nothing
    }
    g.stop();
    g.down(slpd, d_sd);
  });
}

// ---- d8hdisttostrm / d8vdisttostrm (disttostrm.cu): the BFS from the stream cells, one level per launch
namespace {
long long g_dts_levels = 0;
// the frontier list (listA, one 4-byte entry per strip cell), the level bounds and the block counter (listB), the append / consume
// counters (d_ctr[37], [38])
int dts_bufs(td_ctx* ctx, const Strip& s, td::DtsBufs* b) {
  TD_CUDA(ctx->listA.ensure(sizeof(unsigned) * (size_t)s.cells()));
  TD_CUDA(ctx->listB.ensure(sizeof(unsigned long long) * (td::DTS_BATCH + 3)));
  b->list = ctx->listA.as<unsigned>();
  b->ctr = ctx->d_ctr + 37;
  b->bounds = ctx->listB.as<unsigned long long>();
  b->blkdone = reinterpret_cast<unsigned*>(b->bounds + td::DTS_BATCH + 2);
  return TD_OK;
}
}  // namespace
int td_disttostrm_seed_dev(td_ctx* ctx, const int16_t* p, const int32_t* src, float* dist, uint8_t* code, td_strip s, int thresh, int16_t p_nodata,
                           int32_t src_nodata, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !p || !src || !dist || !code || Strip(s).cells() >= (1ll << 32)) {
    td::set_error("td_disttostrm_seed_dev: bad arguments (a strip holds fewer than 2^32 cells, halo rows and padding included)");
    return TD_ERR_ARG;
  }
  td::DtsBufs b;
  if (int rc = dts_bufs(ctx, Strip(s), &b)) return rc;
  return td::dts_seed(p, src, dist, code, Strip(s), thresh, p_nodata, src_nodata, b, (cudaStream_t)stream);
}
int td_disttostrm_levels_dev(td_ctx* ctx, int vertical, const uint8_t* code, const float* fel, const float* rowdist, float* dist, td_strip s,
                             unsigned long long* cells, long long* levels, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !code || !dist || (vertical ? !fel : !rowdist) || Strip(s).cells() >= (1ll << 32) || ctx->listA.cap < sizeof(unsigned) * (size_t)Strip(s).cells()) {
    td::set_error("td_disttostrm_levels_dev: bad arguments (td_disttostrm_seed_dev of this strip comes first, on this context)");
    return TD_ERR_ARG;
  }
  td::DtsBufs b;
  if (int rc = dts_bufs(ctx, Strip(s), &b)) return rc;
  int dev = 0, sms = 1;
  TD_CUDA(cudaGetDevice(&dev));
  TD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return td::dts_levels(vertical != 0, code, fel, rowdist, dist, Strip(s), b, sms * 4, cells, levels, (cudaStream_t)stream);
}
long long td_disttostrm_last_levels(void) { return g_dts_levels; }
}  // extern "C"

namespace {
// src/D8HDistToStrm.cpp:57-226 / src/D8VDistToStrm.cpp:58-240 on one strip
int dts_host(const char* who, bool vertical, const int16_t* p, const float* fel, const int32_t* src, float* dist, int nx, int ny, int16_t p_nodata,
             int32_t src_nodata, int thresh, const double* dxc, const double* dyc) {
  const bool ok = p && src && dist && (vertical ? fel != nullptr : (dxc && dyc));
  return host_call(who, ok && (long long)(ny + 2) * td_pitch_for(nx) < (1ll << 32), nx, ny, [&](HostGrid& g) {
    const float* d_rd = vertical ? nullptr : g.dist(dxc, dyc);
    const int16_t* d_p = g.in(p);
    const int32_t* d_src = g.in(src);
    const float* d_fel = vertical ? g.in(fel) : nullptr;
    float* d_dist = g.alloc<float>();
    uint8_t* d_code = g.alloc<uint8_t>();
    g.start();
    HG_TD(td_disttostrm_seed_dev(g.ctx, d_p, d_src, d_dist, d_code, g.s, thresh, p_nodata, src_nodata, g.st));
    long long levels = 0;
    HG_TD(td_disttostrm_levels_dev(g.ctx, vertical, d_code, d_fel, d_rd, d_dist, g.s, nullptr, &levels, g.st));
    g_dts_levels = levels;
    g.stop();
    g.down(dist, d_dist);
  }, " (fewer than 2^32 strip cells)");
}
}  // namespace

extern "C" {
int td_d8hdisttostrm_host(const int16_t* p, const int32_t* src, float* dist, int nx, int ny, int16_t p_nodata, int32_t src_nodata, int thresh,
                          const double* dxc, const double* dyc) {
  return dts_host("td_d8hdisttostrm_host", false, p, nullptr, src, dist, nx, ny, p_nodata, src_nodata, thresh, dxc, dyc);
}
int td_d8vdisttostrm_host(const int16_t* p, const float* fel, const int32_t* src, float* dist, int nx, int ny, int16_t p_nodata, int32_t src_nodata,
                          int thresh) {
  return dts_host("td_d8vdisttostrm_host", true, p, fel, src, dist, nx, ny, p_nodata, src_nodata, thresh, nullptr, nullptr);
}
}  // extern "C"

// ---- dinfdistdown (dinfdistdown.cu): Kahn's algorithm over the D-infinity receivers, one level per launch on the disttostrm frontier
namespace {
long long g_ddd_levels = 0;
bool ddd_strip_ok(const td_strip& s) { return Strip(s).cells() < (1ll << 32); }
const char* const DDD_STRIP = " (a strip holds fewer than 2^32 cells, halo rows and padding included)";
// theta_ready: the caller has loaded the strip's row angles into ctx->theta (upload_theta_from_host)
int ddd_seed(td_ctx* ctx, const float* ang, const int16_t* src, float* dd, float* dd2, uint8_t* state, td_strip s, float ang_nodata,
             const double* dxc, const double* dyc, bool theta_ready, cudaStream_t st) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !ang || !src || !dd || !state || (!theta_ready && (!dxc || !dyc)) || !ddd_strip_ok(s)) {
    td::set_error(std::string("td_dinfdistdown_seed_dev: bad arguments") + DDD_STRIP);
    return TD_ERR_ARG;
  }
  if (!theta_ready) { if (int rc = upload_theta(ctx, dxc, dyc, s.ny, ctx->theta, st)) return rc; }
  td::DtsBufs b;
  if (int rc = dts_bufs(ctx, Strip(s), &b)) return rc;
  td::DddArgs A{};
  A.theta = ctx->theta.as<double>();
  A.val = dd;
  A.val2 = dd2;
  A.state = state;
  return td::ddd_seed(ang, src, ang_nodata, A, Strip(s), b, st);
}
}  // namespace

extern "C" {
int td_dinfdistdown_seed_dev(td_ctx* ctx, const float* ang, const int16_t* src, float* dd, float* dd2, uint8_t* state, td_strip s, float ang_nodata,
                             const double* dxc, const double* dyc, void* stream) {
  return ddd_seed(ctx, ang, src, dd, dd2, state, s, ang_nodata, dxc, dyc, false, (cudaStream_t)stream);
}
int td_dinfdistdown_levels_dev(td_ctx* ctx, int typemethod, int statmethod, const float* ang, const float* fel, const float* w, const float* rowdist,
                               float* dd, float* dd2, uint8_t* state, td_strip s, float fel_nodata, float w_nodata, int concheck, int* halo_out,
                               unsigned long long* cells, long long* levels, void* stream) {
  if (int rc = check_strip(s)) return rc;
  const bool ok = ctx && ang && dd && state && typemethod >= 0 && typemethod <= 3 && statmethod >= 0 && statmethod <= 2 &&
                  (typemethod == 1 || rowdist) && (typemethod == 0 || fel) && (typemethod != 2 || dd2) && ddd_strip_ok(s) &&
                  (halo_out || (!s.has_top && !s.has_bot)) &&
                  ctx->listA.cap >= sizeof(unsigned) * (size_t)Strip(s).cells();
  if (!ok) {
    td::set_error(std::string("td_dinfdistdown_levels_dev: bad arguments (td_dinfdistdown_seed_dev of this strip comes first, on this "
                              "context)") + DDD_STRIP);
    return TD_ERR_ARG;
  }
  td::DtsBufs b;
  if (int rc = dts_bufs(ctx, Strip(s), &b)) return rc;
  td::DddArgs A{ang, fel, typemethod == 1 ? nullptr : w, rowdist, ctx->theta.as<double>(), dd, typemethod == 2 ? dd2 : nullptr, state, halo_out,
                fel_nodata, w_nodata, concheck == 1};
  int dev = 0, sms = 1;
  TD_CUDA(cudaGetDevice(&dev));
  TD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return td::ddd_levels(typemethod, statmethod, A, Strip(s), b, sms * 4, cells, levels, (cudaStream_t)stream);
}
int td_dinfdistdown_edge_dev(td_ctx* ctx, uint8_t* state, const int* dec_top, const int* dec_bot, td_strip s, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !state || !ddd_strip_ok(s) || ctx->listA.cap < sizeof(unsigned) * (size_t)Strip(s).cells()) {
    td::set_error("td_dinfdistdown_edge_dev: bad arguments (td_dinfdistdown_seed_dev of this strip comes first, on this context)");
    return TD_ERR_ARG;
  }
  td::DtsBufs b;
  if (int rc = dts_bufs(ctx, Strip(s), &b)) return rc;
  return td::ddd_edge(state, dec_top, dec_bot, Strip(s), b, (cudaStream_t)stream);
}
int td_dinfdistdown_pythagoras_dev(td_ctx* ctx, float* dd, const float* dd2, td_strip s, void* stream) {
  if (int rc = check_strip(s)) return rc;
  if (!ctx || !dd || !dd2) {
    td::set_error("td_dinfdistdown_pythagoras_dev: bad arguments");
    return TD_ERR_ARG;
  }
  return td::ddd_pythagoras(dd, dd2, Strip(s), (cudaStream_t)stream);
}
long long td_dinfdistdown_last_levels(void) { return g_ddd_levels; }

// src/DinfDistDown.cpp:66-90 on one strip
int td_dinfdistdown_host(const float* ang, const float* fel, const float* w, const int16_t* src, float* dd, int nx, int ny, float ang_nodata,
                         float fel_nodata, float w_nodata, const double* dxc, const double* dyc, int statmethod, int typemethod, int concheck) {
  const bool ok = ang && src && dd && dxc && dyc && (typemethod == 0 || fel) && typemethod >= 0 && typemethod <= 3 && statmethod >= 0 &&
                  statmethod <= 2;
  return host_call("td_dinfdistdown_host", ok && (long long)(ny + 2) * td_pitch_for(nx) < (1ll << 32), nx, ny, [&](HostGrid& g) {
    HG_TD(upload_theta_from_host(g.ctx, dxc, dyc, ny, g.ctx->theta, g.st));
    const float* d_rd = typemethod == 1 ? nullptr : g.dist(dxc, dyc);
    const float* d_ang = g.in(ang);
    const float* d_fel = typemethod == 0 ? nullptr : g.in(fel);
    const float* d_w = typemethod == 1 ? nullptr : g.in(w);
    const int16_t* d_src = g.in(src);
    float* d_dd = g.alloc<float>();
    float* d_dd2 = typemethod == 2 ? g.alloc<float>() : nullptr;
    uint8_t* d_state = g.alloc<uint8_t>();
    g.start();
    HG_TD(ddd_seed(g.ctx, d_ang, d_src, d_dd, d_dd2, d_state, g.s, ang_nodata, nullptr, nullptr, true, g.st));
    long long levels = 0;
    HG_TD(td_dinfdistdown_levels_dev(g.ctx, typemethod, statmethod, d_ang, d_fel, d_w, d_rd, d_dd, d_dd2, d_state, g.s, fel_nodata, w_nodata,
                                     concheck, nullptr, nullptr, &levels, g.st));
    if (typemethod == 2) HG_TD(td_dinfdistdown_pythagoras_dev(g.ctx, d_dd, d_dd2, g.s, g.st));
    g_ddd_levels = levels;
    g.stop();
    g.down(dd, d_dd);
  }, " (fewer than 2^32 strip cells)");
}

// aread8 + areadinf of one DEM in ONE call with the copies overlapped with the kernels: three streams — host -> device (p, then
// ang), compute (aread8 as soon as p has arrived, areadinf as soon as ang has and aread8 is done), device -> host (ad8 while
// areadinf runs, then sca).  Same kernels, same results as td_aread8_host followed by td_area_host (no weights, no outlets).
// Host rasters should be pinned (cudaHostAlloc / cudaHostRegister) — pageable memory makes the copies synchronous.
int td_contributing_areas_host(const int16_t* p, const float* ang, float* ad8, float* sca, int nx, int ny, int16_t p_nodata, float ang_nodata,
                               const double* dxc, const double* dyc, int contcheck) {
  if (int rc = need_device()) return rc;
  if (!p || !ang || !ad8 || !sca || !dxc || !dyc || nx <= 0 || ny <= 0) { td::set_error("td_contributing_areas_host: bad arguments"); return TD_ERR_ARG; }
  HostGrid g(nx, ny);            // its io slots and its timer; the streams are this call's own
  td_ctx* ctx = g.ctx;
  const td_strip s = g.s;
  int16_t* d_p; float *d_ad8, *d_ang, *d_sca;
  try { d_p = g.alloc<int16_t>(); d_ad8 = g.alloc<float>(); d_ang = g.alloc<float>(); d_sca = g.alloc<float>(); } catch (const Stop& e) { return e.rc; }
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
  g.timer.start(S.run);
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
  td::set_compute_seconds(g.timer.stop(S.run));
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
  return host_call("td_area_host", ang && sca && dxc && dyc, nx, ny, [&](HostGrid& g) {
    float* d_ang = g.alloc<float>();
    float* d_sca = g.alloc<float>();
    const double *d_dx, *d_dy;
    g.cell_sizes(dxc, dyc, &d_dx, &d_dy);
    g.up(d_ang, ang);
    const float* d_w = g.in(w);
    g.start();
    HG_TD(td_area_deps_dev(g.ctx, d_ang, d_sca, g.s, ang_nodata, d_dx, d_dy, g.st));
    g.restrict_to(outlet_cols, outlet_rows, nout);
    HG_TD(td_area_sweep_dev(g.ctx, d_ang, d_w, d_sca, g.s, w != nullptr, contcheck, d_dx, g.st));
    g.stop();
    g.down(sca, d_sca);
  });
}

}  // extern "C"
