// File-level entry points: the five reference library functions re-created behind the
// C ABI (reference prototypes: src/flood.h, src/d8.h:7, src/tardemlib.h:70, src/aread8.h:3,
// src/areadinf.h:2).  Each one reads its rasters with the tiffIO contract, runs the
// device path through the host-grid level of this library and writes the outputs with
// the reference's data types and nodata values (SURVEY.md 8(b) "File contract").
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <chrono>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "../../include/taudem_b200.h"
#include "mgpu.h"
#include "tiff_io.h"

namespace td { void set_error(const std::string& msg); }

namespace {
double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct Input {
  tdio::Raster r;
  std::string path;
  std::vector<double> dxc, dyc;
  int nx = 0, ny = 0;
  // mirrors tiffIO::tiffIO (src/tiffIO.cpp:54-185) including its console messages
  int open(const char* p) {
    path = p;
    std::string err;
    if (!r.open(p, &err)) {
      printf("Error opening file %s.\n", p);
      fflush(stdout);
      td::set_error(err);
      return TD_ERR_IO;
    }
    printf("Input file %s has %s coordinate system.\n", p, r.geo().is_geographic ? "geographic" : "projected");
    nx = (int)r.width(); ny = (int)r.height();
    r.cell_sizes(&dxc, &dyc);
    return TD_OK;
  }
  template <typename T> int read(std::vector<T>* out, tdio::DType t) {
    out->resize((size_t)nx * ny);
    std::string err;
    // stream by row blocks to bound the decode scratch
    const long blk = std::max<long>(1, (64l << 20) / ((long)nx * 4));
    for (long y = 0; y < ny; y += blk) {
      const long n = std::min<long>(blk, ny - y);
      if (!r.read(0, y, n, nx, out->data() + (size_t)y * nx, t, &err)) { td::set_error(err); printf("Error reading %s: %s\n", path.c_str(), err.c_str()); return TD_ERR_IO; }
    }
    return TD_OK;
  }
};

// tiffIO copy-constructor + write (src/tiffIO.cpp:187-243, 263-428): same size and
// georeferencing as `like`, given type and nodata, name by the reference's extension rule.
template <typename T>
int write_like(const char* name, const Input& like, tdio::DType t, double nodata, const T* data) {
  const std::string path = tdio::output_path_rule(name);
  const size_t dot = path.rfind('.');
  const std::string ext = dot == std::string::npos ? "" : path.substr(dot);
  if (ext != ".tif" && ext != ".tiff") {
    printf("GDAL driver is not available\n");   // only the GTiff driver exists here (src/tiffIO.cpp:309-314)
    td::set_error("only .tif/.tiff outputs are supported: " + path);
    return TD_ERR_DRIVER;
  }
  const int cellbytes = t == tdio::DT_I16 ? 2 : 4;
  const double fileGB = (double)cellbytes * like.nx * (double)like.ny / 1000000000.0;
  if (fileGB > 4.0) printf("Setting BIGTIFF, File: %s, Anticipated size (GB):%.2f\n", path.c_str(), fileGB);
  tdio::Writer w;
  std::string err;
  // LZW like the reference's GTiff creation options (src/tiffIO.cpp:316-318); TAUDEM_B200_COMPRESS = NONE | DEFLATE | LZW overrides
  const char* comp_env = getenv("TAUDEM_B200_COMPRESS");
  int comp = 5;
  if (comp_env && strcmp(comp_env, "NONE") == 0) comp = 1;
  if (comp_env && strcmp(comp_env, "DEFLATE") == 0) comp = 8;
  if (!w.create(path, like.nx, like.ny, t, nodata, like.r.geo(), comp, &err) || !w.write_rows(0, like.ny, data, &err) || !w.close(&err)) {
    printf("Error writing %s: %s\n", path.c_str(), err.c_str());
    td::set_error(err);
    return TD_ERR_IO;
  }
  return TD_OK;
}

template <typename T>
int write_like(const char* name, const Input& like, tdio::DType t, double nodata, const std::vector<T>& data) {
  return write_like(name, like, t, nodata, data.data());
}

// TAUDEM_B200_GPUS=N (N > 1): the reference's `mpiexec -n N <tool>` — one forked process per GPU, each with its row strip
// (mgpu.cu).  pitremove / d8flowdir / dinfflowdir / peukerdouglas (mgpu_flow): the ranks read their rows of the DEM, the parent
// writes the rasters
int flow_multi_gpu(int tool, int world, const Input& dem, const char* demfile, const char* maskfile, int use_mask, int four, const char* out0file,
                   const char* out1file, double t0, double t1, const float* par = nullptr) {
  const size_t n = (size_t)dem.nx * dem.ny;
  const size_t b0 = n * (tool == 1 || tool == 3 ? 2 : 4), b1 = (tool == 0 || tool == 3) ? 0 : n * 4;
  void* out0 = td::mgpu_alloc_shared(b0);
  float* out1 = b1 ? (float*)td::mgpu_alloc_shared(b1) : nullptr;
  if (!out0 || (b1 && !out1)) { td::mgpu_free_shared(out0, b0); td::mgpu_free_shared(out1, b1); td::set_error("cannot map the shared output rasters"); return TD_ERR_IO; }
  td::MgpuFlowJob J;
  J.tool = tool; J.demfile = demfile; J.maskfile = maskfile; J.use_mask = use_mask; J.four = four; J.nx = dem.nx; J.ny = dem.ny; J.out0 = out0; J.out1 = out1;
  if (par) for (int i = 0; i < 3; ++i) J.par[i] = par[i];
  double secs = 0.; int rounds = 0; long long left = 0;
  int rc = td::mgpu_flow(J, world, &secs, &rounds, &left);
  const double t2 = now();
  const char* name = tool == 0 ? "PitRemove" : tool == 1 ? "D8FlowDir" : tool == 2 ? "DinfFlowDir" : "PeukerDouglas";
  double t3 = t2, t4 = t2;
  if (rc) printf("%s device error: %s\n", name, td_last_error());
  else if (tool == 0) { rc = write_like(out0file, dem, tdio::DT_F32, (double)-3.0e38f, (const float*)out0); t3 = t4 = now(); }
  else if (tool == 3) { rc = write_like(out0file, dem, tdio::DT_I16, (double)(int16_t)-2, (const int16_t*)out0); t3 = t4 = now(); }
  else {
    rc = write_like(out1file, dem, tdio::DT_F32, (double)-1.0f, (const float*)out1);            // slope first, like the reference
    t3 = now();
    if (!rc) rc = tool == 1 ? write_like(out0file, dem, tdio::DT_I16, (double)(short)-32768, (const int16_t*)out0)
                            : write_like(out0file, dem, tdio::DT_F32, (double)-3.402823466e+38F, (const float*)out0);
    t4 = now();
  }
  td::mgpu_free_shared(out0, b0); td::mgpu_free_shared(out1, b1);
  if (rc) return rc;
  // (the ranks read their rows inside what is reported as compute time; the header pass is the read time)
  if (tool == 0)
    printf("Processes: %d\nHeader read time: %f\nData read time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", world, t1 - t0, 0.0, t2 - t1, t3 - t2, t3 - t0);
  else if (tool == 3)
    printf("Processors: %d\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", world, t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  else
    printf("Processors: %d\nHeader read time: %f\nData read time: %f\nCompute Slope time: %f\nWrite Slope time: %f\nResolve Flat time: %f\nWrite Flat time: %f\nTotal time: %f\n",
           world, t1 - t0, 0.0, t2 - t1, t3 - t2, 0.0, t4 - t3, t4 - t0);
  if (tool == 3) printf("Device compute time: %f\nExchange rounds: %d\n", secs, rounds);
  else printf("Device compute time: %f\nExchange rounds: %d\nFlat cells left: %lld\n", secs, rounds, left);
  return TD_OK;
}

// the CUDA context comes up on a helper thread while the tool opens and reads its rasters
struct Warmup {
  std::thread th;
  Warmup() : th([] { td_warmup(); }) {}
  void join() { if (th.joinable()) th.join(); }
  ~Warmup() { join(); }
};

void nodata_msgs(double nd, const char* what, double cast) {
  // createpart.h:57-85 prints these two lines for every partition created from a file
  printf("Nodata value input to create partition from file: %lf\n", nd);
  printf("Nodata value recast to %s used in partition raster: %s\n", what, std::to_string(cast).c_str());
}
// one more grid of a sibling tool: open, compare with the direction grid (companion_open); then read it
int companion_open(const Input& a, Input& g, const char* file, tdio::DType dt, const char* type, const char* what = "companion grid does not match") {
  if (int rc = g.open(file)) return rc;
  if (!tdio::compare_rasters(a.r, a.path, g.r, g.path)) { printf("File sizes do not match\n%s\n", file); td::set_error(what); return TD_ERR_MISMATCH; }
  if (dt == tdio::DT_F32) nodata_msgs(g.r.nodata(), type, (float)g.r.nodata());
  else if (dt == tdio::DT_I32) nodata_msgs(g.r.nodata(), type, (int32_t)g.r.nodata());
  else nodata_msgs(g.r.nodata(), type, (int16_t)g.r.nodata());
  return TD_OK;
}
template <typename T>
int companion(Input& a, Input& g, const char* file, std::vector<T>* data, tdio::DType dt, const char* type) {
  if (int rc = companion_open(a, g, file, dt, type)) return rc;
  return g.read(data, dt);
}

// TAUDEM_B200_GPUS=N for the sweep tools (mgpu_sibling): the ranks read their rows of every input, the parent writes the outputs (mapping
// slot, file, type, nodata) in the order the single-GPU run writes them; nproc_label heads the process count's line
bool use_multi_gpu(const Input& in, int useOutlets) { return td::mgpu_world() > 1 && useOutlets != 1 && in.ny >= td::mgpu_world(); }
struct SibOut { int slot; const char* file; tdio::DType t; double nodata; };
int sibling_multi_gpu(td::MgpuSibJob& J, const Input& like, const std::vector<SibOut>& outs, double t0, const char* name,
                      const char* nproc_label = "Processors") {
  const int world = td::mgpu_world();
  const size_t n = (size_t)like.nx * like.ny;
  size_t bytes[3] = {0, 0, 0};
  for (const SibOut& o : outs) bytes[o.slot] = n * (o.t == tdio::DT_I16 ? 2 : 4);
  bool mapped = true;
  for (int i = 0; i < 3; ++i) if (bytes[i]) { J.out[i] = td::mgpu_alloc_shared(bytes[i]); mapped = mapped && J.out[i]; }
  auto unmap = [&]() { for (int i = 0; i < 3; ++i) td::mgpu_free_shared(J.out[i], bytes[i]); };
  if (!mapped) { unmap(); td::set_error("cannot map the shared output rasters"); return TD_ERR_IO; }
  J.nx = like.nx; J.ny = like.ny;
  const double t1 = now();
  double secs = 0.; int rounds = 0;
  int rc = td::mgpu_sibling(J, world, &secs, &rounds);
  const double t2 = now();
  if (rc) printf("%s device error: %s\n", name, td_last_error());
  for (const SibOut& o : outs) {
    if (rc) break;
    rc = o.t == tdio::DT_I16 ? write_like(o.file, like, o.t, o.nodata, (const int16_t*)J.out[o.slot]) : write_like(o.file, like, o.t, o.nodata, (const float*)J.out[o.slot]);
  }
  const double t3 = now();
  unmap();
  if (rc) return rc;
  // (the ranks read their rows inside what is reported as compute time: Read time is the header pass)
  printf("%s: %d\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", nproc_label, world, t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\nExchange rounds: %d\n", secs, rounds);
  return TD_OK;
}

}  // namespace

extern "C" {

int td_nameadd(char* full, const char* arg, const char* suff) {
  // suffix goes before the extension; the original extension is kept unless the suffix has its own
  const char* ext = strrchr(arg, '.');
  const char* extsuff = strrchr(suff, '.');
  if (!ext) { sprintf(full, "%s%s", arg, suff); return (int)strlen(arg); }
  const size_t nmain = strlen(arg) - strlen(ext);
  memcpy(full, arg, nmain);
  full[nmain] = 0;
  strcat(full, suff);
  if (!extsuff) strcat(full, ext);
  return (int)nmain;
}

int td_raster_info(const char* path, int* nx, int* ny, double* nodata, int* has_nodata, double* dx, double* dy, int* is_geographic,
                   int* bits, int* sample_format) try {
  tdio::Raster r; std::string err;
  if (!r.open(path, &err)) { td::set_error(err); return TD_ERR_IO; }
  if (nx) *nx = (int)r.width();
  if (ny) *ny = (int)r.height();
  if (nodata) *nodata = r.nodata();
  if (has_nodata) *has_nodata = r.has_nodata();
  if (dx) *dx = fabs(r.geo().gt[1]);
  if (dy) *dy = fabs(r.geo().gt[5]);
  if (is_geographic) *is_geographic = r.geo().is_geographic;
  if (bits) *bits = r.bits();
  if (sample_format) *sample_format = r.sample_format();
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}
int td_raster_read(const char* path, int dtype, void* dest, int nx, int ny) try {
  tdio::Raster r; std::string err;
  if (!r.open(path, &err)) { td::set_error(err); return TD_ERR_IO; }
  if ((int)r.width() != nx || (int)r.height() != ny) { td::set_error("td_raster_read: size mismatch"); return TD_ERR_ARG; }
  if (!r.read(0, 0, ny, nx, dest, (tdio::DType)dtype, &err)) { td::set_error(err); return TD_ERR_IO; }
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}
int td_raster_cell_sizes(const char* path, double* dxc, double* dyc, int ny) try {
  tdio::Raster r; std::string err;
  if (!r.open(path, &err)) { td::set_error(err); return TD_ERR_IO; }
  if ((int)r.height() != ny) { td::set_error("td_raster_cell_sizes: size mismatch"); return TD_ERR_ARG; }
  std::vector<double> x, y; r.cell_sizes(&x, &y);
  memcpy(dxc, x.data(), sizeof(double) * ny); memcpy(dyc, y.data(), sizeof(double) * ny);
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}
int td_raster_write(const char* path, int dtype, const void* src, int nx, int ny, double nodata, const char* like_path, double dx,
                    double dy, int compression) try {
  tdio::GeoInfo geo; std::string err;
  if (like_path) {
    tdio::Raster r;
    if (!r.open(like_path, &err)) { td::set_error(err); return TD_ERR_IO; }
    geo = r.geo();
  } else {
    geo.gt[0] = 0; geo.gt[1] = dx; geo.gt[2] = 0; geo.gt[3] = dy * ny; geo.gt[4] = 0; geo.gt[5] = -dy;
  }
  tdio::Writer w;
  const bool force_big = (compression & 0x100) != 0;     // bit 8: write BigTIFF regardless of size (tests)
  compression &= 0xff;
  if (!w.create(path, nx, ny, (tdio::DType)dtype, nodata, geo, compression, &err, force_big) || !w.write_rows(0, ny, src, &err) || !w.close(&err)) {
    td::set_error(err); return TD_ERR_IO;
  }
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

int td_flood(const char* demfile, const char* felfile, const char* sfdrfile, int usesfdr, int verbose, int is_4Point, int use_mask,
             const char* maskfile) try {
  (void)sfdrfile; (void)usesfdr;     // not implemented by the reference either (src/PitRemovemn.cpp:143)
  printf("PitRemove version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input dem;
  if (int rc = dem.open(demfile)) return rc;
  Input mask;
  if (use_mask) {
    if (int rc = mask.open(maskfile)) return rc;
    if (!tdio::compare_rasters(dem.r, dem.path, mask.r, mask.path)) {
      printf("Error using mask file.\n");
      td::set_error("depression mask does not match the DEM");
      return TD_ERR_ARG;
    }
  }
  const double t1 = now();
  std::vector<float> z; std::vector<int16_t> m;
  nodata_msgs(dem.r.nodata(), "float", (float)dem.r.nodata());
  if (td::mgpu_world() > 1 && dem.ny >= td::mgpu_world()) {
    if (use_mask) nodata_msgs(mask.r.nodata(), "int16_t", (int16_t)mask.r.nodata());
    return flow_multi_gpu(0, td::mgpu_world(), dem, demfile, maskfile, use_mask, is_4Point, felfile, nullptr, t0, t1);
  }
  if (int rc = dem.read(&z, tdio::DT_F32)) return rc;
  if (use_mask) { nodata_msgs(mask.r.nodata(), "int16_t", (int16_t)mask.r.nodata()); if (int rc = mask.read(&m, tdio::DT_I16)) return rc; }
  const double t2 = now();
  if (verbose) {
    printf("Data read\n");
    printf("Midpoint of partition: 0, nxm: %d, nym: %d, value: %f\n", dem.nx / 2, dem.ny / 2, z[(size_t)(dem.ny / 2) * dem.nx + dem.nx / 2]);
  }
  std::vector<float> fel((size_t)dem.nx * dem.ny);
  if (int rc = td_flood_host(z.data(), fel.data(), use_mask ? m.data() : nullptr, dem.nx, dem.ny, (float)dem.r.nodata(), is_4Point)) {
    printf("PitRemove device error: %s\n", td_last_error());
    return rc;
  }
  const double t3 = now();
  const float felNodata = -3.0e38f;
  if (int rc = write_like(felfile, dem, tdio::DT_F32, (double)felNodata, fel)) return rc;
  const double t4 = now();
  printf("Processes: 1\nHeader read time: %f\nData read time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1,
         t3 - t2, t4 - t3, t4 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

int td_setdird8(const char* demfile, const char* pointfile, const char* slopefile, const char* flowfile, int useflowfile) try {
  (void)flowfile; (void)useflowfile;   // -sfdr is accepted and functionally dead in the reference (src/d8.cpp:243-267)
  printf("D8FlowDir version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input dem;
  if (int rc = dem.open(demfile)) return rc;
  const double t1 = now();
  std::vector<float> z;
  nodata_msgs(dem.r.nodata(), "float", (float)dem.r.nodata());
  if (td::mgpu_world() > 1 && dem.ny >= td::mgpu_world()) return flow_multi_gpu(1, td::mgpu_world(), dem, demfile, nullptr, 0, 0, pointfile, slopefile, t0, t1);
  if (int rc = dem.read(&z, tdio::DT_F32)) return rc;
  const double t2 = now();
  std::vector<int16_t> p((size_t)dem.nx * dem.ny);
  std::vector<float> sd8((size_t)dem.nx * dem.ny);
  if (int rc = td_setdird8_host(z.data(), p.data(), sd8.data(), dem.nx, dem.ny, (float)dem.r.nodata(), dem.dxc.data(), dem.dyc.data())) {
    printf("D8FlowDir device error: %s\n", td_last_error());
    return rc;
  }
  const double t3 = now();
  if (int rc = write_like(slopefile, dem, tdio::DT_F32, (double)-1.0f, sd8)) return rc;
  const double t4 = now();
  if (int rc = write_like(pointfile, dem, tdio::DT_I16, (double)(short)-32768, p)) return rc;
  const double t5 = now();
  printf("Processors: 1\nHeader read time: %f\nData read time: %f\nCompute Slope time: %f\nWrite Slope time: %f\nResolve Flat time: %f\nWrite Flat time: %f\nTotal time: %f\n",
         t1 - t0, t2 - t1, t3 - t2, t4 - t3, 0.0, t5 - t4, t5 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

int td_setdir(const char* demfile, const char* angfile, const char* slopefile, const char* flowfile, int useflowfile) try {
  (void)flowfile; (void)useflowfile;
  printf("DinfFlowDir version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input dem;
  if (int rc = dem.open(demfile)) return rc;
  const double t1 = now();
  std::vector<float> z;
  nodata_msgs(dem.r.nodata(), "float", (float)dem.r.nodata());
  if (td::mgpu_world() > 1 && dem.ny >= td::mgpu_world()) return flow_multi_gpu(2, td::mgpu_world(), dem, demfile, nullptr, 0, 0, angfile, slopefile, t0, t1);
  if (int rc = dem.read(&z, tdio::DT_F32)) return rc;
  const double t2 = now();
  std::vector<float> ang((size_t)dem.nx * dem.ny), slp((size_t)dem.nx * dem.ny);
  if (int rc = td_setdir_host(z.data(), ang.data(), slp.data(), dem.nx, dem.ny, (float)dem.r.nodata(), dem.dxc.data(), dem.dyc.data())) {
    printf("DinfFlowDir device error: %s\n", td_last_error());
    return rc;
  }
  const double t3 = now();
  if (int rc = write_like(slopefile, dem, tdio::DT_F32, (double)-1.0f, slp)) return rc;
  const double t4 = now();
  const float missing = -3.402823466e+38F;   // MISSINGFLOAT (src/commonLib.h:80)
  if (int rc = write_like(angfile, dem, tdio::DT_F32, (double)missing, ang)) return rc;
  const double t5 = now();
  printf("Processors: 1\nHeader read time: %f\nData read time: %f\nCompute Slope time: %f\nWrite Slope time: %f\nResolve Flat time: %f\nWrite Flat time: %f\nTotal time: %f\n",
         t1 - t0, t2 - t1, t3 - t2, t4 - t3, 0.0, t5 - t4, t5 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// readoutlets + geoToGlobalXY (src/aread8.cpp:112-120,179-188, src/tiffIO.cpp:580-588): outlet points -> grid cells
static int outlet_cells(const char* datasrc, const char* lyrname, int uselyrname, int lyrno, const Input& in, std::vector<int>* cols,
                        std::vector<int>* rows) {
  int n = 0;
  if (int rc = td_outlets_read(datasrc, lyrname, uselyrname, lyrno, nullptr, nullptr, 0, &n)) { printf("Read outlets error: %s\n", td_last_error()); return rc; }
  std::vector<double> x(n > 0 ? n : 1), y(n > 0 ? n : 1);
  if (int rc = td_outlets_read(datasrc, lyrname, uselyrname, lyrno, x.data(), y.data(), n, &n)) return rc;
  const tdio::GeoInfo& g = in.r.geo();
  const double xleft = g.gt[0], ytop = g.gt[3], dlon = std::fabs(g.gt[1]), dlat = std::fabs(g.gt[5]);
  cols->resize(n); rows->resize(n);
  for (int i = 0; i < n; ++i) {
    (*cols)[i] = (int)((x[i] - xleft) / dlon);
    (*rows)[i] = (int)((ytop - y[i]) / dlat);
  }
  return TD_OK;
}

int td_aread8(const char* pfile, const char* afile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, const char* wfile,
              int useOutlets, int usew, int contcheck) try {
  {  // src/aread8.cpp:62-71
    FILE* fp = fopen(pfile, "r");
    if (!fp) { fprintf(stderr, "Error: Input file %s does not exist.\n", pfile); td::set_error("input file does not exist"); return TD_ERR_IO; }
    fclose(fp);
  }
  printf("AreaD8 version %s\n", td_version());
  const double t0 = now();
  Input p;
  if (int rc = p.open(pfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, p, &ocols, &orows)) return rc; }
  std::vector<int16_t> dir;
  nodata_msgs(p.r.nodata(), "int16_t", (int16_t)p.r.nodata());
  if (use_multi_gpu(p, useOutlets)) {
    Input w;
    if (usew) { if (int rc = companion_open(p, w, wfile, tdio::DT_F32, "float", "weight grid does not match")) return rc; }
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::AREAD8; J.dirfile = pfile; J.in[0] = usew ? wfile : nullptr; J.contcheck = contcheck;
    return sibling_multi_gpu(J, p, {{0, afile, tdio::DT_F32, (double)-1.0f}}, t0, "AreaD8", "Number of Processes");
  }
  Warmup warm;
  if (int rc = p.read(&dir, tdio::DT_I16)) return rc;
  Input w; std::vector<float> wg;
  if (usew) {
    if (int rc = w.open(wfile)) return rc;
    if (!tdio::compare_rasters(p.r, p.path, w.r, w.path)) { printf("File sizes do not match\n%s\n", wfile); td::set_error("weight grid does not match"); return TD_ERR_MISMATCH; }
    nodata_msgs(w.r.nodata(), "float", (float)w.r.nodata());
    if (int rc = w.read(&wg, tdio::DT_F32)) return rc;
  }
  const double t1 = now();
  std::unique_ptr<float[]> ad8(new float[(size_t)p.nx * p.ny]);      // not zero-filled: every cell is written by the download
  warm.join();
  if (int rc = td_aread8_outlets_host(dir.data(), usew ? wg.data() : nullptr, ad8.get(), p.nx, p.ny, (int16_t)p.r.nodata(),
                                      usew ? (float)w.r.nodata() : 0.f, contcheck, ocols.data(), orows.data(),
                                      useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("AreaD8 device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(afile, p, tdio::DT_F32, (double)-1.0f, (const float*)ad8.get())) return rc;
  const double t3 = now();
  printf("Number of Processes: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

int td_area(const char* angfile, const char* scafile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, const char* wfile,
            int useOutlets, int usew, int contcheck) try {
  printf("AreaDinf version %s\n", td_version());
  const double t0 = now();
  Input a;
  if (int rc = a.open(angfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, a, &ocols, &orows)) return rc; }
  std::vector<float> ang;
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  if (use_multi_gpu(a, useOutlets)) {
    Input w;
    if (usew) {
      if (int rc = w.open(wfile)) return rc;
      if (!tdio::compare_rasters(a.r, a.path, w.r, w.path)) { td::set_error("weight grid does not match"); return TD_ERR_ARG; }
      nodata_msgs(w.r.nodata(), "float", (float)w.r.nodata());
    }
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::AREADINF; J.dirfile = angfile; J.in[0] = usew ? wfile : nullptr; J.contcheck = contcheck;
    return sibling_multi_gpu(J, a, {{0, scafile, tdio::DT_F32, (double)-1.0f}}, t0, "AreaDinf");
  }
  Warmup warm;
  if (int rc = a.read(&ang, tdio::DT_F32)) return rc;
  Input w; std::vector<float> wg;
  if (usew) {
    if (int rc = w.open(wfile)) return rc;
    if (!tdio::compare_rasters(a.r, a.path, w.r, w.path)) { td::set_error("weight grid does not match"); return TD_ERR_ARG; }   // src/areadinf.cpp:132
    nodata_msgs(w.r.nodata(), "float", (float)w.r.nodata());
    if (int rc = w.read(&wg, tdio::DT_F32)) return rc;
  }
  const double t1 = now();
  std::unique_ptr<float[]> sca(new float[(size_t)a.nx * a.ny]);
  warm.join();
  if (int rc = td_area_outlets_host(ang.data(), usew ? wg.data() : nullptr, sca.get(), a.nx, a.ny, (float)a.r.nodata(),
                                    usew ? (float)w.r.nodata() : 0.f, a.dxc.data(), a.dyc.data(), contcheck, ocols.data(), orows.data(),
                                    useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("AreaDinf device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(scafile, a, tdio::DT_F32, (double)-1.0f, (const float*)sca.get())) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  // a malformed file (or an allocation failure) must not unwind through the C ABI
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}


// src/D8flowpathextremeup.cpp:58-285
int td_d8flowpathextremeup(const char* pfile, const char* safile, const char* ssafile, int usemax, const char* datasrc, const char* lyrname,
                           int uselyrname, int lyrno, int useOutlets, int contcheck) try {
  printf("D8FlowPathExtremeUp version %s\n", td_version());
  const double t0 = now();
  Input p;
  if (int rc = p.open(pfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, p, &ocols, &orows)) return rc; }
  std::vector<int16_t> dir;
  nodata_msgs(p.r.nodata(), "int16_t", (int16_t)p.r.nodata());
  if (use_multi_gpu(p, useOutlets)) {
    Input a;
    if (int rc = companion_open(p, a, safile, tdio::DT_F32, "float", "value grid does not match")) return rc;
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::EXTREMEUP; J.dirfile = pfile; J.in[0] = safile; J.usemax = usemax; J.contcheck = contcheck;
    return sibling_multi_gpu(J, p, {{0, ssafile, tdio::DT_F32, (double)-3.4028234663852886e38f}}, t0, "D8FlowPathExtremeUp");
  }
  if (int rc = p.read(&dir, tdio::DT_I16)) return rc;
  Input a; std::vector<float> sa;
  if (int rc = a.open(safile)) return rc;
  if (!tdio::compare_rasters(p.r, p.path, a.r, a.path)) { printf("File sizes do not match\n%s\n", safile); td::set_error("value grid does not match"); return TD_ERR_MISMATCH; }
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  if (int rc = a.read(&sa, tdio::DT_F32)) return rc;
  const double t1 = now();
  std::vector<float> ssa((size_t)p.nx * p.ny);
  if (int rc = td_d8flowpathextremeup_host(dir.data(), sa.data(), ssa.data(), p.nx, p.ny, (int16_t)p.r.nodata(), usemax, contcheck, ocols.data(),
                                           orows.data(), useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("D8FlowPathExtremeUp device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(ssafile, p, tdio::DT_F32, (double)-3.4028234663852886e38f, ssa)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/Threshold.cpp:48-162
// gridnet (src/gridnet.cpp:55-500)
int td_gridnet(const char* pfile, const char* plenfile, const char* tlenfile, const char* gordfile, const char* maskfile, const char* datasrc,
               const char* lyrname, int uselyrname, int lyrno, int useMask, int useOutlets, int thresh) try {
  printf("GridNet version %s\n", td_version());
  const double t0 = now();
  Input p;
  if (int rc = p.open(pfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, p, &ocols, &orows)) return rc; }
  std::vector<int16_t> dir;
  nodata_msgs(p.r.nodata(), "int16_t", (int16_t)p.r.nodata());
  if (use_multi_gpu(p, useOutlets)) {
    Input m;
    if (useMask == 1) { if (int rc = companion_open(p, m, maskfile, tdio::DT_I32, "int32_t", "mask grid does not match")) return rc; }
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::GRIDNET; J.dirfile = pfile; J.in[0] = useMask == 1 ? maskfile : nullptr; J.thresh = thresh;
    return sibling_multi_gpu(J, p, {{2, gordfile, tdio::DT_I16, -1.0}, {0, plenfile, tdio::DT_F32, (double)-1.0f}, {1, tlenfile, tdio::DT_F32, (double)-1.0f}},
                             t0, "GridNet");
  }
  if (int rc = p.read(&dir, tdio::DT_I16)) return rc;
  Input m; std::vector<int32_t> mask;
  if (useMask == 1) {
    if (int rc = m.open(maskfile)) return rc;
    if (!tdio::compare_rasters(p.r, p.path, m.r, m.path)) { printf("File sizes do not match\n%s\n", maskfile); td::set_error("mask grid does not match"); return TD_ERR_MISMATCH; }
    nodata_msgs(m.r.nodata(), "int32_t", (int32_t)m.r.nodata());
    if (int rc = m.read(&mask, tdio::DT_I32)) return rc;
  }
  const double t1 = now();
  const size_t n = (size_t)p.nx * p.ny;
  std::vector<float> plen(n), tlen(n); std::vector<int16_t> gord(n);
  if (int rc = td_gridnet_host(dir.data(), useMask == 1 ? mask.data() : nullptr, thresh, plen.data(), tlen.data(), gord.data(), p.nx, p.ny, (int16_t)p.r.nodata(),
                               p.dxc.data(), p.dyc.data(), ocols.data(), orows.data(), useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("GridNet device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(gordfile, p, tdio::DT_I16, -1.0, gord)) return rc;
  if (int rc = write_like(plenfile, p, tdio::DT_F32, (double)-1.0f, plen)) return rc;
  if (int rc = write_like(tlenfile, p, tdio::DT_F32, (double)-1.0f, tlen)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// dmarea (src/dinfdecayaccum.cpp:61-323)
int td_dmarea(const char* angfile, const char* adecfile, const char* dmfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
              const char* wfile, int useOutlets, int usew, int contcheck) try {
  printf("DinfDecayAccum version %s\n", td_version());
  const double t0 = now();
  Input a;
  if (int rc = a.open(angfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, a, &ocols, &orows)) return rc; }
  std::vector<float> ang, dm, wg;
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  if (use_multi_gpu(a, useOutlets)) {
    Input d, w;
    if (int rc = companion_open(a, d, dmfile, tdio::DT_F32, "float", "decay multiplier grid does not match")) return rc;
    if (usew) { if (int rc = companion_open(a, w, wfile, tdio::DT_F32, "float", "weight grid does not match")) return rc; }
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::DECAY; J.dirfile = angfile; J.in[0] = dmfile; J.in[1] = usew ? wfile : nullptr; J.contcheck = contcheck;
    return sibling_multi_gpu(J, a, {{0, adecfile, tdio::DT_F32, (double)-3.4028234663852886e38f}}, t0, "DinfDecayAccum");
  }
  if (int rc = a.read(&ang, tdio::DT_F32)) return rc;
  Input d;
  if (int rc = d.open(dmfile)) return rc;
  if (!tdio::compare_rasters(a.r, a.path, d.r, d.path)) { printf("File sizes do not match\n%s\n", dmfile); td::set_error("decay multiplier grid does not match"); return TD_ERR_MISMATCH; }
  nodata_msgs(d.r.nodata(), "float", (float)d.r.nodata());
  if (int rc = d.read(&dm, tdio::DT_F32)) return rc;
  Input w;
  if (usew) {
    if (int rc = w.open(wfile)) return rc;
    if (!tdio::compare_rasters(a.r, a.path, w.r, w.path)) { printf("File sizes do not match\n%s\n", wfile); td::set_error("weight grid does not match"); return TD_ERR_MISMATCH; }
    nodata_msgs(w.r.nodata(), "float", (float)w.r.nodata());
    if (int rc = w.read(&wg, tdio::DT_F32)) return rc;
  }
  const double t1 = now();
  std::vector<float> out((size_t)a.nx * a.ny);
  if (int rc = td_dinfdecayaccum_host(ang.data(), dm.data(), usew ? wg.data() : nullptr, out.data(), a.nx, a.ny, (float)a.r.nodata(), (float)d.r.nodata(),
                                      a.dxc.data(), a.dyc.data(), contcheck, ocols.data(), orows.data(), useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("DinfDecayAccum device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(adecfile, a, tdio::DT_F32, (double)-3.4028234663852886e38f, out)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/DinfConcLimAccum.cpp:61-347
int td_dsllarea(const char* angfile, const char* ctptfile, const char* dmfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
                const char* qfile, const char* dgfile, int useOutlets, int contcheck, float cSol) try {
  printf("DinfConcLimAccum version %s\n", td_version());
  const double t0 = now();
  Input a;
  if (int rc = a.open(angfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, a, &ocols, &orows)) return rc; }
  std::vector<float> ang, dm, q;
  std::vector<int16_t> dg;
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  if (use_multi_gpu(a, useOutlets)) {
    Input d, g, qq;
    if (int rc = companion_open(a, d, dmfile, tdio::DT_F32, "float")) return rc;
    if (int rc = companion_open(a, g, dgfile, tdio::DT_I16, "int16_t")) return rc;
    if (int rc = companion_open(a, qq, qfile, tdio::DT_F32, "float")) return rc;
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::CONCLIM; J.dirfile = angfile; J.in[0] = dmfile; J.in[1] = qfile; J.in[2] = dgfile; J.csol = cSol; J.contcheck = contcheck;
    return sibling_multi_gpu(J, a, {{0, ctptfile, tdio::DT_F32, (double)-3.4028234663852886e38f}}, t0, "DinfConcLimAccum");
  }
  if (int rc = a.read(&ang, tdio::DT_F32)) return rc;
  Input d, g, qq;
  if (int rc = companion(a, d, dmfile, &dm, tdio::DT_F32, "float")) return rc;
  if (int rc = companion(a, g, dgfile, &dg, tdio::DT_I16, "int16_t")) return rc;
  if (int rc = companion(a, qq, qfile, &q, tdio::DT_F32, "float")) return rc;
  const double t1 = now();
  std::vector<float> out((size_t)a.nx * a.ny);
  if (int rc = td_dinfconclimaccum_host(ang.data(), dm.data(), q.data(), dg.data(), out.data(), a.nx, a.ny, (float)a.r.nodata(), (float)d.r.nodata(),
                                        (float)qq.r.nodata(), cSol, a.dxc.data(), a.dyc.data(), contcheck, ocols.data(), orows.data(),
                                        useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("DinfConcLimAccum device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(ctptfile, a, tdio::DT_F32, (double)-3.4028234663852886e38f, out)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/DinfTransLimAccum.cpp:61-394
int td_tlaccum(const char* angfile, const char* tsupfile, const char* tcfile, const char* tlafile, const char* depfile, const char* cinfile,
               const char* coutfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, int useOutlets, int usec, int contcheck) try {
  printf("DinfTransLimAccum version %s\n", td_version());
  const double t0 = now();
  Input a;
  if (int rc = a.open(angfile)) return rc;
  std::vector<int> ocols, orows;
  if (useOutlets == 1) { if (int rc = outlet_cells(datasrc, lyrname, uselyrname, lyrno, a, &ocols, &orows)) return rc; }
  std::vector<float> ang, tsup, tc, cin;
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  if (use_multi_gpu(a, useOutlets)) {
    Input ts, tcc, ci;
    if (int rc = companion_open(a, ts, tsupfile, tdio::DT_F32, "float")) return rc;
    if (int rc = companion_open(a, tcc, tcfile, tdio::DT_F32, "float")) return rc;
    if (usec == 1) { if (int rc = companion_open(a, ci, cinfile, tdio::DT_F32, "float")) return rc; }
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::TRANSLIM; J.dirfile = angfile; J.in[0] = tsupfile; J.in[1] = tcfile; J.in[2] = usec == 1 ? cinfile : nullptr; J.contcheck = contcheck;
    std::vector<SibOut> outs = {{0, tlafile, tdio::DT_F32, (double)-3.4028234663852886e38f}, {1, depfile, tdio::DT_F32, (double)-3.4028234663852886e38f}};
    if (usec == 1) outs.push_back({2, coutfile, tdio::DT_F32, (double)-3.4028234663852886e38f});
    return sibling_multi_gpu(J, a, outs, t0, "DinfTransLimAccum");
  }
  if (int rc = a.read(&ang, tdio::DT_F32)) return rc;
  Input ts, tcc, ci;
  if (int rc = companion(a, ts, tsupfile, &tsup, tdio::DT_F32, "float")) return rc;
  if (int rc = companion(a, tcc, tcfile, &tc, tdio::DT_F32, "float")) return rc;
  if (usec == 1) { if (int rc = companion(a, ci, cinfile, &cin, tdio::DT_F32, "float")) return rc; }
  const double t1 = now();
  const size_t n = (size_t)a.nx * a.ny;
  std::vector<float> tla(n), dep(n), cout(usec == 1 ? n : 0);
  if (int rc = td_dinftranslimaccum_host(ang.data(), tsup.data(), tc.data(), usec == 1 ? cin.data() : nullptr, tla.data(), dep.data(),
                                         usec == 1 ? cout.data() : nullptr, a.nx, a.ny, (float)a.r.nodata(), (float)ts.r.nodata(), (float)tcc.r.nodata(),
                                         usec == 1 ? (float)ci.r.nodata() : 0.f, a.dxc.data(), a.dyc.data(), contcheck, ocols.data(), orows.data(),
                                         useOutlets == 1 ? (int)ocols.size() : -1)) {
    printf("DinfTransLimAccum device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(tlafile, a, tdio::DT_F32, (double)-3.4028234663852886e38f, tla)) return rc;
  if (int rc = write_like(depfile, a, tdio::DT_F32, (double)-3.4028234663852886e38f, dep)) return rc;
  if (usec == 1) { if (int rc = write_like(coutfile, a, tdio::DT_F32, (double)-3.4028234663852886e38f, cout)) return rc; }
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

int td_threshold(const char* ssafile, const char* srcfile, const char* maskfile, float thresh, int usemask) try {
  printf("Threshold version %s\n", td_version());
  const double t0 = now();
  Input a;
  if (int rc = a.open(ssafile)) return rc;
  std::vector<float> ssa;
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  if (int rc = a.read(&ssa, tdio::DT_F32)) return rc;
  Input m; std::vector<float> mask;
  if (usemask == 1) {
    if (int rc = m.open(maskfile)) return rc;
    if (!tdio::compare_rasters(a.r, a.path, m.r, m.path)) { td::set_error("mask grid does not match"); return TD_ERR_ARG; }   // src/Threshold.cpp:89
    nodata_msgs(m.r.nodata(), "float", (float)m.r.nodata());
    if (int rc = m.read(&mask, tdio::DT_F32)) return rc;
  }
  const double t1 = now();
  std::vector<int16_t> src((size_t)a.nx * a.ny);
  if (int rc = td_threshold_host(ssa.data(), usemask == 1 ? mask.data() : nullptr, src.data(), a.nx, a.ny, thresh, (float)a.r.nodata())) {
    printf("Threshold device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(srcfile, a, tdio::DT_I16, (double)(int16_t)-32768, src)) return rc;
  const double t3 = now();
  printf("Compute time: %f\n", t2 - t1);
  printf("Read time: %f\nWrite time: %f\nTotal time: %f\nDevice compute time: %f\n", t1 - t0, t3 - t2, t3 - t0, td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/TWI.cpp:47-155
int td_twigrid(const char* slopefile, const char* areafile, const char* twifile) try {
  printf("Topographic Wetness Index version %s\n", td_version());
  const double t0 = now();
  Input sl;
  if (int rc = sl.open(slopefile)) return rc;
  std::vector<float> slp;
  nodata_msgs(sl.r.nodata(), "float", (float)sl.r.nodata());
  if (int rc = sl.read(&slp, tdio::DT_F32)) return rc;
  Input ar; std::vector<float> sca;
  if (int rc = ar.open(areafile)) return rc;
  if (!tdio::compare_rasters(sl.r, sl.path, ar.r, ar.path)) { td::set_error("area grid does not match"); return TD_ERR_ARG; }   // src/TWI.cpp:88
  nodata_msgs(ar.r.nodata(), "float", (float)ar.r.nodata());
  if (int rc = ar.read(&sca, tdio::DT_F32)) return rc;
  const double t1 = now();
  std::vector<float> twi((size_t)sl.nx * sl.ny);
  if (int rc = td_twi_host(slp.data(), sca.data(), twi.data(), sl.nx, sl.ny, (float)sl.r.nodata(), (float)ar.r.nodata())) {
    printf("TWI device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(twifile, sl, tdio::DT_F32, (double)-1.0f, twi)) return rc;
  const double t3 = now();
  printf("Compute time: %f\n", t2 - t1);
  printf("Read time: %f\nWrite time: %f\nTotal time: %f\nDevice compute time: %f\n", t1 - t0, t3 - t2, t3 - t0, td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/SlopeArea.cpp:52-156 and src/SlopeAreaRatio.cpp:49-150: two float rasters in, one out (nodata -1), same messages
static int two_in_one_out(int which, const char* banner, const char* slopefile, const char* scafile, const char* outfile, const float* par) {
  printf("%s version %s\n", banner, td_version());
  const double t0 = now();
  Input sl;
  if (int rc = sl.open(slopefile)) return rc;
  std::vector<float> slp;
  nodata_msgs(sl.r.nodata(), "float", (float)sl.r.nodata());
  if (int rc = sl.read(&slp, tdio::DT_F32)) return rc;
  Input ar; std::vector<float> sca;
  if (int rc = ar.open(scafile)) return rc;
  if (!tdio::compare_rasters(sl.r, sl.path, ar.r, ar.path)) { td::set_error("area grid does not match"); return 1; }   // `return 1`, src/SlopeArea.cpp:89
  nodata_msgs(ar.r.nodata(), "float", (float)ar.r.nodata());
  if (int rc = ar.read(&sca, tdio::DT_F32)) return rc;
  const double t1 = now();
  std::vector<float> out((size_t)sl.nx * sl.ny);
  const int rc = which == 0 ? td_slopearea_host(slp.data(), sca.data(), out.data(), sl.nx, sl.ny, par[0], par[1])
                            : td_slopearearatio_host(slp.data(), sca.data(), out.data(), sl.nx, sl.ny, (float)ar.r.nodata());
  if (rc) { printf("%s device error: %s\n", banner, td_last_error()); return rc; }
  const double t2 = now();
  if (int rc2 = write_like(outfile, sl, tdio::DT_F32, (double)-1.0f, out)) return rc2;
  const double t3 = now();
  printf("Compute time: %f\n", t2 - t1);
  printf("Read time: %f\nWrite time: %f\nTotal time: %f\nDevice compute time: %f\n", t1 - t0, t3 - t2, t3 - t0, td_last_compute_seconds());
  return TD_OK;
}
int td_slopearea(const char* slopefile, const char* scafile, const char* safile, const float* p) try {
  if (!p) { td::set_error("td_slopearea: the exponents are missing"); return TD_ERR_ARG; }
  return two_in_one_out(0, "SlopeArea", slopefile, scafile, safile, p);
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}
int td_atanbgrid(const char* slopefile, const char* areafile, const char* atanbfile) try {
  return two_in_one_out(1, "SlopeAreaRatio", slopefile, areafile, atanbfile, nullptr);
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/PeukerDouglas.cpp:54-241: fel in, ss out (int16, nodata tag -2, georeference of fel); TAUDEM_B200_GPUS=N runs it on N row strips
int td_peukerdouglas(const char* felfile, const char* ssfile, const float* p) try {
  if (!p) { td::set_error("td_peukerdouglas: the weights are missing"); return TD_ERR_ARG; }
  printf("PeukerDouglas version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input fel;
  if (int rc = fel.open(felfile)) return rc;
  nodata_msgs(fel.r.nodata(), "float", (float)fel.r.nodata());
  if (td::mgpu_world() > 1 && fel.ny >= td::mgpu_world())
    return flow_multi_gpu(3, td::mgpu_world(), fel, felfile, nullptr, 0, 0, ssfile, nullptr, t0, now(), p);
  Warmup warm;
  std::vector<float> z;
  if (int rc = fel.read(&z, tdio::DT_F32)) return rc;
  warm.join();
  const double t1 = now();
  std::vector<int16_t> ss((size_t)fel.nx * fel.ny);
  if (int rc = td_peukerdouglas_host(z.data(), ss.data(), fel.nx, fel.ny, (float)fel.r.nodata(), p)) {
    printf("PeukerDouglas device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(ssfile, fel, tdio::DT_I16, (double)(int16_t)-2, ss)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/LengthArea.cpp:51-149: plen (float) and ad8 (read as int32) in, ss out (int16, nodata -32768, georeference of ad8)
int td_lengtharea(const char* plenfile, const char* ad8file, const char* ssfile, const float* p) try {
  if (!p) { td::set_error("td_lengtharea: the coefficient and exponent are missing"); return TD_ERR_ARG; }
  printf("LengthArea version %s\n", td_version());
  const double t0 = now();
  Input pl;
  if (int rc = pl.open(plenfile)) return rc;
  std::vector<float> plen;
  nodata_msgs(pl.r.nodata(), "float", (float)pl.r.nodata());
  if (int rc = pl.read(&plen, tdio::DT_F32)) return rc;
  Input ad; std::vector<int32_t> ad8;
  if (int rc = ad.open(ad8file)) return rc;
  if (!tdio::compare_rasters(pl.r, pl.path, ad.r, ad.path)) { td::set_error("ad8 grid does not match"); return TD_ERR_ARG; }   // `return 1`, src/LengthArea.cpp:88
  nodata_msgs(ad.r.nodata(), "int32_t", (int32_t)ad.r.nodata());
  if (int rc = ad.read(&ad8, tdio::DT_I32)) return rc;
  const double t1 = now();
  std::vector<int16_t> ss((size_t)pl.nx * pl.ny);
  if (int rc = td_lengtharea_host(plen.data(), ad8.data(), ss.data(), pl.nx, pl.ny, p[0], p[1])) {
    printf("LengthArea device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  printf("Compute time: %f\n", t2 - t1);
  if (int rc = write_like(ssfile, ad, tdio::DT_I16, (double)(int16_t)-32768, ss)) return rc;
  const double t3 = now();
  printf("Read time: %f\nWrite time: %f\nTotal time: %f\nDevice compute time: %f\n", t1 - t0, t3 - t2, t3 - t0, td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/SlopeAveDown.cpp:59-330: fel and p in, slpd out (float32, nodata MISSINGFLOAT, the georeference of p).  The distances use fel's
// per-row cell sizes; niter uses its header cell sizes, dxA / dyA = |dxc| / |dyc| of the middle row (src/tiffIO.cpp:155).
// TAUDEM_B200_GPUS=N runs it on N row strips.
int td_sloped(const char* pfile, const char* felfile, const char* slpdfile, double dn) try {
  printf("SlopeAveDown version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input z;
  if (int rc = z.open(felfile)) return rc;
  nodata_msgs(z.r.nodata(), "float", (float)z.r.nodata());
  Input p;
  if (int rc = companion_open(z, p, pfile, tdio::DT_I16, "int16_t", "flow direction grid does not match")) return rc;
  const double dxA = fabs(z.dxc[z.ny / 2]), dyA = fabs(z.dyc[z.ny / 2]);
  int niter = 0;
  if (int rc = td_slopeavedown_niter(dn, dxA, dyA, &niter)) return rc;
  if (td::mgpu_world() > 1 && z.ny >= td::mgpu_world()) {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::SLOPEAVEDOWN; J.dirfile = pfile; J.in[0] = felfile; J.dn = dn; J.niter = niter;
    return sibling_multi_gpu(J, p, {{0, slpdfile, tdio::DT_F32, (double)-3.4028234663852886e38f}}, t0, "SlopeAveDown");
  }
  Warmup warm;
  std::vector<float> fel;
  std::vector<int16_t> dir;
  if (int rc = z.read(&fel, tdio::DT_F32)) return rc;
  if (int rc = p.read(&dir, tdio::DT_I16)) return rc;
  warm.join();
  const double t1 = now();
  std::vector<float> sd((size_t)z.nx * z.ny);
  if (int rc = td_slopeavedown_host(fel.data(), dir.data(), sd.data(), z.nx, z.ny, (float)z.r.nodata(), (int16_t)p.r.nodata(), z.dxc.data(), z.dyc.data(),
                                    dxA, dyA, dn)) {
    printf("SlopeAveDown device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(slpdfile, p, tdio::DT_F32, (double)-3.4028234663852886e38f, sd)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/flowdircond.cpp:56-236: p (int16) and z (float) in, zfdc out (float32, the nodata value and the georeference of z: the reference
// writes zIO.getNodata(), the double of z's header).
// TAUDEM_B200_GPUS=N runs it on N row strips.
int td_flowdircond(const char* pfile, const char* zfile, const char* zfdcfile) try {
  printf("FlowDirCond version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input p;
  if (int rc = p.open(pfile)) return rc;
  nodata_msgs(p.r.nodata(), "int16_t", (int16_t)p.r.nodata());
  Input z;
  if (int rc = companion_open(p, z, zfile, tdio::DT_F32, "float", "elevation grid does not match")) return rc;
  if (use_multi_gpu(p, 0)) {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::FLOWDIRCOND; J.dirfile = pfile; J.in[0] = zfile;
    return sibling_multi_gpu(J, z, {{0, zfdcfile, tdio::DT_F32, z.r.nodata()}}, t0, "FlowDirCond");
  }
  Warmup warm;
  std::vector<int16_t> dir;
  std::vector<float> zv;
  if (int rc = p.read(&dir, tdio::DT_I16)) return rc;
  if (int rc = z.read(&zv, tdio::DT_F32)) return rc;
  warm.join();
  const double t1 = now();
  std::vector<float> out((size_t)p.nx * p.ny);
  if (int rc = td_flowdircond_host(dir.data(), zv.data(), out.data(), p.nx, p.ny, (int16_t)p.r.nodata(), (float)z.r.nodata())) {
    printf("FlowDirCond device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(zfdcfile, z, tdio::DT_F32, z.r.nodata(), out)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/RetlimFlow.cpp:53-240: ang, wg and rc (float) in, qrl out (float32, nodata MISSINGFLOAT, the georeference of rc).  The shares use
// ang's per-row cell sizes.  TAUDEM_B200_GPUS=N runs it on N row strips.
int td_retlimro(const char* angfile, const char* wgfile, const char* rcfile, const char* qrlfile) try {
  printf("Retention limited flow accumulation version %s\n", td_version());
  fflush(stdout);
  const double t0 = now();
  Input a;
  if (int rc = a.open(angfile)) return rc;
  nodata_msgs(a.r.nodata(), "float", (float)a.r.nodata());
  Input w, r;
  if (int rc = companion_open(a, w, wgfile, tdio::DT_F32, "float", "weight grid does not match")) return rc;
  if (int rc = companion_open(a, r, rcfile, tdio::DT_F32, "float", "retention capacity grid does not match")) return rc;
  if (use_multi_gpu(a, 0)) {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::RETLIMFLOW; J.dirfile = angfile; J.in[0] = wgfile; J.in[1] = rcfile;
    return sibling_multi_gpu(J, r, {{0, qrlfile, tdio::DT_F32, (double)-3.4028234663852886e38f}}, t0, "RetlimFlow");
  }
  Warmup warm;
  std::vector<float> ang, wg, rcv;
  if (int rc = a.read(&ang, tdio::DT_F32)) return rc;
  if (int rc = w.read(&wg, tdio::DT_F32)) return rc;
  if (int rc = r.read(&rcv, tdio::DT_F32)) return rc;
  warm.join();
  const double t1 = now();
  std::vector<float> out((size_t)a.nx * a.ny);
  if (int rc = td_retlimflow_host(ang.data(), wg.data(), rcv.data(), out.data(), a.nx, a.ny, (float)a.r.nodata(), (float)w.r.nodata(), (float)r.r.nodata(),
                                  a.dxc.data(), a.dyc.data())) {
    printf("RetlimFlow device error: %s\n", td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc = write_like(qrlfile, r, tdio::DT_F32, (double)-3.4028234663852886e38f, out)) return rc;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}

// src/D8HDistToStrm.cpp:57-226 / src/D8VDistToStrm.cpp:58-240: p (int16), fel (float, vertical only) and src (int32) in, dist out
// (float32, nodata MISSINGFLOAT, the georeference of p).  The horizontal distances use p's per-row cell sizes.  TAUDEM_B200_GPUS=N
// runs it on N row strips.
static int disttostrm(bool vertical, const char* pfile, const char* felfile, const char* srcfile, const char* distfile, int thresh) try {
  const char* name = vertical ? "D8VDistToStrm" : "D8HDistToStrm";
  printf("%s version %s\n", name, td_version());
  fflush(stdout);
  const double t0 = now();
  Input p;
  if (int rc = p.open(pfile)) return rc;
  nodata_msgs(p.r.nodata(), "int16_t", (int16_t)p.r.nodata());
  Input z, g;
  if (vertical) { if (int rc = companion_open(p, z, felfile, tdio::DT_F32, "float", "elevation grid does not match")) return rc; }
  if (int rc = companion_open(p, g, srcfile, tdio::DT_I32, "int32_t", "stream raster does not match")) return rc;
  if (use_multi_gpu(p, 0)) {
    td::MgpuSibJob J;
    J.tool = vertical ? td::MgpuSibJob::D8VDIST : td::MgpuSibJob::D8HDIST; J.dirfile = pfile; J.in[0] = srcfile; J.in[1] = vertical ? felfile : nullptr;
    J.thresh = thresh;
    return sibling_multi_gpu(J, p, {{0, distfile, tdio::DT_F32, (double)-3.4028234663852886e38f}}, t0, name);
  }
  Warmup warm;
  std::vector<int16_t> dir;
  std::vector<float> fel;
  std::vector<int32_t> src;
  if (int rc = p.read(&dir, tdio::DT_I16)) return rc;
  if (vertical) { if (int rc = z.read(&fel, tdio::DT_F32)) return rc; }
  if (int rc = g.read(&src, tdio::DT_I32)) return rc;
  warm.join();
  const double t1 = now();
  std::vector<float> dist((size_t)p.nx * p.ny);
  const int rc = vertical ? td_d8vdisttostrm_host(dir.data(), fel.data(), src.data(), dist.data(), p.nx, p.ny, (int16_t)p.r.nodata(), (int32_t)g.r.nodata(), thresh)
                          : td_d8hdisttostrm_host(dir.data(), src.data(), dist.data(), p.nx, p.ny, (int16_t)p.r.nodata(), (int32_t)g.r.nodata(), thresh,
                                                  p.dxc.data(), p.dyc.data());
  if (rc) {
    printf("%s device error: %s\n", name, td_last_error());
    return rc;
  }
  const double t2 = now();
  if (int rc2 = write_like(distfile, p, tdio::DT_F32, (double)-3.4028234663852886e38f, dist)) return rc2;
  const double t3 = now();
  printf("Processors: 1\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t1 - t0, t2 - t1, t3 - t2, t3 - t0);
  printf("Device compute time: %f\n", td_last_compute_seconds());
  return TD_OK;
} catch (const std::exception& e) {
  td::set_error(std::string("exception: ") + e.what());
  return TD_ERR_IO;
}
int td_distgrid(const char* pfile, const char* srcfile, const char* distfile, int thresh) {
  return disttostrm(false, pfile, nullptr, srcfile, distfile, thresh);
}
int td_d8vdistdown(const char* pfile, const char* felfile, const char* srcfile, const char* distfile, int thresh) {
  return disttostrm(true, pfile, felfile, srcfile, distfile, thresh);
}

}  // extern "C"
