// File-level entry points: one per executable, each re-creating the reference tool's library function behind the C ABI.  An entry
// point states what is particular to its tool (its inputs, outputs, report, multi-GPU job and one compute call of the host-grid level
// of this library); run() does the rest: it opens and checks the rasters with the tiffIO contract, runs the device path on one GPU or
// on TAUDEM_B200_GPUS forked ranks (mgpu.cu), and writes the outputs with the reference's data types and nodata values (SURVEY.md
// 8(b) "File contract").
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <chrono>
#include <functional>
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

constexpr double MISSINGFLOAT = (double)-3.402823466e+38F;   // src/commonLib.h:80
const tdio::DType F32 = tdio::DT_F32, I16 = tdio::DT_I16, I32 = tdio::DT_I32;

// every C-ABI entry point of this file: a malformed file (or an allocation failure) must not unwind through the C ABI
template <class F> int guarded(F&& body) {
  try {
    return body();
  } catch (const std::exception& e) {
    td::set_error(std::string("exception: ") + e.what());
    return TD_ERR_IO;
  }
}

struct Input {
  tdio::Raster r;
  tdio::DType t = F32;
  std::string path;
  std::vector<double> dxc, dyc;
  int nx = 0, ny = 0;
  std::unique_ptr<char[]> data;    // the cells once read; NULL for an input that is not used
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
  // createpart.h:57-85 prints these two lines for every partition created from a file
  void nodata_msgs() const {
    const double nd = r.nodata(), cast = t == F32 ? (double)(float)nd : t == I32 ? (double)(int32_t)nd : (double)(int16_t)nd;
    printf("Nodata value input to create partition from file: %lf\n", nd);
    printf("Nodata value recast to %s used in partition raster: %s\n", t == F32 ? "float" : t == I32 ? "int32_t" : "int16_t",
           std::to_string(cast).c_str());
  }
  int read() {
    const size_t eb = tdio::dtype_bytes(t);
    data.reset(new char[(size_t)nx * ny * eb]);      // not zero-filled: every cell is read or the read fails
    std::string err;
    // stream by row blocks to bound the decode scratch
    const long blk = std::max<long>(1, (64l << 20) / ((long)nx * 4));
    for (long y = 0; y < ny; y += blk) {
      const long n = std::min<long>(blk, ny - y);
      if (!r.read(0, y, n, nx, data.get() + (size_t)y * nx * eb, t, &err)) { td::set_error(err); printf("Error reading %s: %s\n", path.c_str(), err.c_str()); return TD_ERR_IO; }
    }
    return TD_OK;
  }
  template <class T> const T* as() const { return (const T*)data.get(); }
  float fnd() const { return (float)r.nodata(); }
  int16_t snd() const { return (int16_t)r.nodata(); }
};

// tiffIO copy-constructor + write (src/tiffIO.cpp:187-243, 263-428): same size and
// georeferencing as `like`, given type and nodata, name by the reference's extension rule.
int write_like(const char* name, const Input& like, tdio::DType t, double nodata, const void* data) {
  const std::string path = tdio::output_path_rule(name);
  const size_t dot = path.rfind('.');
  const std::string ext = dot == std::string::npos ? "" : path.substr(dot);
  if (ext != ".tif" && ext != ".tiff") {
    printf("GDAL driver is not available\n");   // only the GTiff driver exists here (src/tiffIO.cpp:309-314)
    td::set_error("only .tif/.tiff outputs are supported: " + path);
    return TD_ERR_DRIVER;
  }
  const double fileGB = (double)tdio::dtype_bytes(t) * like.nx * (double)like.ny / 1000000000.0;
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

// the CUDA context comes up on a helper thread while the tool reads its rasters
struct Warmup {
  std::thread th;
  Warmup() : th([] { td_warmup(); }) {}
  void join() { if (th.joinable()) th.join(); }
  ~Warmup() { join(); }
};

// What a companion raster whose size differs from the first input's does, as each reference tool does it
enum Mismatch {
  SIZES,        // prints "File sizes do not match" and the file, returns TD_ERR_MISMATCH (MPI_Abort(MCW, 5) in the reference)
  SILENT,       // returns TD_ERR_ARG
  SILENT_ONE,   // returns 1 (src/SlopeArea.cpp:89)
  MASK_FILE,    // prints "Error using mask file." (src/flood.cpp:79), returns TD_ERR_ARG
};
struct In {
  const char* file;
  tdio::DType t;
  const char* what = "companion grid does not match";   // td::set_error text when the size differs from the first input's
  Mismatch mismatch = SIZES;
  bool used = true;
};
// an output raster: slot = its index in the compute call's and the multi-GPU job's out[]; it takes the size, the georeference and,
// with like_nodata, the nodata value of input `like`
struct Out {
  int slot;
  const char* file;
  tdio::DType t;
  double nodata;
  int like = 0;
  bool like_nodata = false;
  bool used = true;
};
// the timing report: pitremove's, the flow directions' (one time per output written), the sweep tools', and the point-wise tools'
// (Compute time after the write, or before it for lengtharea)
enum Report { PITREMOVE, FLOWDIR, SWEEP, POINT, POINT_COMPUTE_FIRST };
struct Outlets {
  const char* datasrc = nullptr;
  const char* lyrname = nullptr;
  int uselyrname = 0, lyrno = 0, use = 0;
};
struct Tool {
  const char* banner;                 // "<banner> version ..."
  const char* name;                   // "<name> device error: ..."
  std::vector<In> in;                 // in the order they are opened; in[0] gives the grid's size
  std::vector<Out> out;               // in the order they are written
  Report report = SWEEP;
  const char* nproc = "Processors";   // heads the process count's line
  td::MgpuFlowJob* flow = nullptr;    // the rank job, if the tool has one; run() fills in its size and outputs
  td::MgpuSibJob* sib = nullptr;
  Outlets outlets = {};
  bool headers_first = false;         // every header line before the nodata lines, as pitremove (src/flood.cpp:73-77)
  std::function<int(const std::vector<Input>&)> opened;   // a check on the opened inputs before any is read
};
// what the compute call of one GPU sees
struct Grids {
  const std::vector<Input>& in;
  void* const* outp;
  const int* ocols;
  const int* orows;
  int nout;                           // -1 without -o
  template <class T> T* out(int slot) const { return (T*)outp[slot]; }
};

// readoutlets + geoToGlobalXY (src/aread8.cpp:112-120,179-188, src/tiffIO.cpp:580-588): outlet points -> grid cells
int outlet_cells(const Outlets& o, const Input& in, std::vector<int>* cols, std::vector<int>* rows) {
  int n = 0;
  if (int rc = td_outlets_read(o.datasrc, o.lyrname, o.uselyrname, o.lyrno, nullptr, nullptr, 0, &n)) { printf("Read outlets error: %s\n", td_last_error()); return rc; }
  std::vector<double> x(n > 0 ? n : 1), y(n > 0 ? n : 1);
  if (int rc = td_outlets_read(o.datasrc, o.lyrname, o.uselyrname, o.lyrno, x.data(), y.data(), n, &n)) return rc;
  const tdio::GeoInfo& g = in.r.geo();
  const double xleft = g.gt[0], ytop = g.gt[3], dlon = std::fabs(g.gt[1]), dlat = std::fabs(g.gt[5]);
  cols->resize(n); rows->resize(n);
  for (int i = 0; i < n; ++i) {
    (*cols)[i] = (int)((x[i] - xleft) / dlon);
    (*rows)[i] = (int)((ytop - y[i]) / dlat);
  }
  return TD_OK;
}

// the output rasters: anonymous shared mappings that the forked ranks write into, or host memory that is not zero-filled (the
// host-grid calls download every cell of every output they are given)
struct OutBufs {
  void* p[3] = {nullptr, nullptr, nullptr};
  size_t bytes[3] = {0, 0, 0};
  bool shared;
  OutBufs(const std::vector<Out>& outs, size_t cells, bool shared_) : shared(shared_) {
    for (const Out& o : outs) if (o.used) bytes[o.slot] = cells * tdio::dtype_bytes(o.t);
    for (int i = 0; i < 3; ++i) if (bytes[i]) p[i] = shared ? td::mgpu_alloc_shared(bytes[i]) : new char[bytes[i]];
  }
  bool ok() const { for (int i = 0; i < 3; ++i) if (bytes[i] && !p[i]) return false; return true; }
  ~OutBufs() { for (int i = 0; i < 3; ++i) shared ? td::mgpu_free_shared(p[i], bytes[i]) : delete[] (char*)p[i]; }
};

int run(Tool& t, const std::function<int(const Grids&)>& compute) {
  printf("%s version %s\n", t.banner, td_version());
  fflush(stdout);
  const double t0 = now();
  std::vector<Input> in(t.in.size());
  for (size_t k = 0; k < t.in.size(); ++k) {
    const In& s = t.in[k];
    if (!s.used) continue;
    in[k].t = s.t;
    if (int rc = in[k].open(s.file)) return rc;
    if (k && !tdio::compare_rasters(in[0].r, in[0].path, in[k].r, in[k].path)) {
      if (s.mismatch == SIZES) printf("File sizes do not match\n%s\n", s.file);
      if (s.mismatch == MASK_FILE) printf("Error using mask file.\n");
      td::set_error(s.what);
      return s.mismatch == SIZES ? TD_ERR_MISMATCH : s.mismatch == SILENT_ONE ? 1 : TD_ERR_ARG;
    }
    if (!t.headers_first) in[k].nodata_msgs();
  }
  if (t.headers_first) for (size_t k = 0; k < t.in.size(); ++k) if (t.in[k].used) in[k].nodata_msgs();
  if (t.opened) { if (int rc = t.opened(in)) return rc; }
  std::vector<int> ocols, orows;
  if (t.outlets.use == 1) { if (int rc = outlet_cells(t.outlets, in[0], &ocols, &orows)) return rc; }
  const int nx = in[0].nx, ny = in[0].ny, world = td::mgpu_world();
  // TAUDEM_B200_GPUS=N (N > 1): the reference's `mpiexec -n N <tool>`, one forked process per GPU, each with its row strip.  The ranks
  // read their rows inside what is reported as compute time; the header pass is the read time.
  const bool ranks = (t.flow || t.sib) && world > 1 && t.outlets.use != 1 && ny >= world;
  const double t1 = now();
  double t2 = t1, secs = 0.;
  int rounds = 0, rc = 0;
  long long left = 0;
  OutBufs out(t.out, (size_t)nx * ny, ranks);
  if (ranks) {
    if (!out.ok()) { td::set_error("cannot map the shared output rasters"); return TD_ERR_IO; }
    if (t.flow) {
      t.flow->nx = nx; t.flow->ny = ny;
      for (int i = 0; i < 2; ++i) t.flow->out[i] = out.p[i];
      rc = td::mgpu_flow(*t.flow, world, &secs, &rounds, &left);
    } else {
      t.sib->nx = nx; t.sib->ny = ny;
      for (int i = 0; i < 3; ++i) t.sib->out[i] = out.p[i];
      rc = td::mgpu_sibling(*t.sib, world, &secs, &rounds);
    }
  } else {
    Warmup warm;     // only now: the parent must not hold a CUDA context when it forks the ranks
    for (Input& i : in) if (!i.path.empty()) { if (int rc2 = i.read()) return rc2; }
    t2 = now();
    warm.join();
    rc = compute(Grids{in, out.p, ocols.data(), orows.data(), t.outlets.use == 1 ? (int)ocols.size() : -1});
    secs = td_last_compute_seconds();
  }
  const double t3 = now();
  if (rc) { printf("%s device error: %s\n", t.name, td_last_error()); return rc; }
  if (t.report == POINT_COMPUTE_FIRST) printf("Compute time: %f\n", t3 - t2);
  double tw = t3;      // the end of the first write
  int written = 0;
  for (const Out& o : t.out) {
    if (!o.used) continue;
    if (int rc2 = write_like(o.file, in[o.like], o.t, o.like_nodata ? in[o.like].r.nodata() : o.nodata, out.p[o.slot])) return rc2;
    if (written++ == 0) tw = now();
  }
  const double t4 = now();
  const int np = ranks ? world : 1;
  switch (t.report) {
    case PITREMOVE:
      printf("%s: %d\nHeader read time: %f\nData read time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t.nproc, np, t1 - t0, t2 - t1,
             t3 - t2, t4 - t3, t4 - t0);
      break;
    case FLOWDIR:
      printf("%s: %d\nHeader read time: %f\nData read time: %f\nCompute Slope time: %f\nWrite Slope time: %f\nResolve Flat time: %f\nWrite Flat time: %f\n"
             "Total time: %f\n", t.nproc, np, t1 - t0, t2 - t1, t3 - t2, tw - t3, 0.0, t4 - tw, t4 - t0);
      break;
    case SWEEP:
      printf("%s: %d\nRead time: %f\nCompute time: %f\nWrite time: %f\nTotal time: %f\n", t.nproc, np, t2 - t0, t3 - t2, t4 - t3, t4 - t0);
      break;
    case POINT:
      printf("Compute time: %f\n", t3 - t2);
      [[fallthrough]];
    case POINT_COMPUTE_FIRST:
      printf("Read time: %f\nWrite time: %f\nTotal time: %f\n", t2 - t0, t4 - t3, t4 - t0);
      break;
  }
  printf("Device compute time: %f\n", secs);
  if (ranks) printf("Exchange rounds: %d\n", rounds);
  if (ranks && (t.report == PITREMOVE || t.report == FLOWDIR)) printf("Flat cells left: %lld\n", left);
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
                   int* bits, int* sample_format) {
  return guarded([&] {
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
  });
}
int td_raster_read(const char* path, int dtype, void* dest, int nx, int ny) {
  return guarded([&] {
    tdio::Raster r; std::string err;
    if (!r.open(path, &err)) { td::set_error(err); return TD_ERR_IO; }
    if ((int)r.width() != nx || (int)r.height() != ny) { td::set_error("td_raster_read: size mismatch"); return TD_ERR_ARG; }
    if (!r.read(0, 0, ny, nx, dest, (tdio::DType)dtype, &err)) { td::set_error(err); return TD_ERR_IO; }
    return TD_OK;
  });
}
int td_raster_cell_sizes(const char* path, double* dxc, double* dyc, int ny) {
  return guarded([&] {
    tdio::Raster r; std::string err;
    if (!r.open(path, &err)) { td::set_error(err); return TD_ERR_IO; }
    if ((int)r.height() != ny) { td::set_error("td_raster_cell_sizes: size mismatch"); return TD_ERR_ARG; }
    std::vector<double> x, y; r.cell_sizes(&x, &y);
    memcpy(dxc, x.data(), sizeof(double) * ny); memcpy(dyc, y.data(), sizeof(double) * ny);
    return TD_OK;
  });
}
int td_raster_write(const char* path, int dtype, const void* src, int nx, int ny, double nodata, const char* like_path, double dx,
                    double dy, int compression) {
  return guarded([&] {
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
  });
}

// src/flood.cpp
int td_flood(const char* demfile, const char* felfile, const char* sfdrfile, int usesfdr, int verbose, int is_4Point, int use_mask,
             const char* maskfile) {
  (void)sfdrfile; (void)usesfdr;     // not implemented by the reference either (src/PitRemovemn.cpp:143)
  return guarded([&] {
    td::MgpuFlowJob J;
    J.tool = 0; J.demfile = demfile; J.maskfile = maskfile; J.use_mask = use_mask; J.four = is_4Point;
    Tool t{"PitRemove", "PitRemove", {{demfile, F32}, {maskfile, I16, "depression mask does not match the DEM", MASK_FILE, use_mask != 0}},
           {{0, felfile, F32, (double)-3.0e38f}}, PITREMOVE, "Processes", &J};
    t.headers_first = true;
    return run(t, [&](const Grids& g) {
      const Input& dem = g.in[0];
      if (verbose) {
        printf("Data read\n");
        printf("Midpoint of partition: 0, nxm: %d, nym: %d, value: %f\n", dem.nx / 2, dem.ny / 2, dem.as<float>()[(size_t)(dem.ny / 2) * dem.nx + dem.nx / 2]);
      }
      return td_flood_host(dem.as<float>(), g.out<float>(0), g.in[1].as<int16_t>(), dem.nx, dem.ny, dem.fnd(), is_4Point);
    });
  });
}

// src/d8.cpp; the slope is written first, like the reference
int td_setdird8(const char* demfile, const char* pointfile, const char* slopefile, const char* flowfile, int useflowfile) {
  (void)flowfile; (void)useflowfile;   // -sfdr is accepted and functionally dead in the reference (src/d8.cpp:243-267)
  return guarded([&] {
    td::MgpuFlowJob J;
    J.tool = 1; J.demfile = demfile;
    Tool t{"D8FlowDir", "D8FlowDir", {{demfile, F32}}, {{1, slopefile, F32, (double)-1.0f}, {0, pointfile, I16, -32768.0}}, FLOWDIR, "Processors", &J};
    return run(t, [&](const Grids& g) {
      const Input& dem = g.in[0];
      return td_setdird8_host(dem.as<float>(), g.out<int16_t>(0), g.out<float>(1), dem.nx, dem.ny, dem.fnd(), dem.dxc.data(), dem.dyc.data());
    });
  });
}

// src/dinf.cpp
int td_setdir(const char* demfile, const char* angfile, const char* slopefile, const char* flowfile, int useflowfile) {
  (void)flowfile; (void)useflowfile;
  return guarded([&] {
    td::MgpuFlowJob J;
    J.tool = 2; J.demfile = demfile;
    Tool t{"DinfFlowDir", "DinfFlowDir", {{demfile, F32}}, {{1, slopefile, F32, (double)-1.0f}, {0, angfile, F32, MISSINGFLOAT}}, FLOWDIR, "Processors", &J};
    return run(t, [&](const Grids& g) {
      const Input& dem = g.in[0];
      return td_setdir_host(dem.as<float>(), g.out<float>(0), g.out<float>(1), dem.nx, dem.ny, dem.fnd(), dem.dxc.data(), dem.dyc.data());
    });
  });
}

// src/aread8.cpp
int td_aread8(const char* pfile, const char* afile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, const char* wfile,
              int useOutlets, int usew, int contcheck) {
  return guarded([&] {
    {  // src/aread8.cpp:62-71
      FILE* fp = fopen(pfile, "r");
      if (!fp) { fprintf(stderr, "Error: Input file %s does not exist.\n", pfile); td::set_error("input file does not exist"); return TD_ERR_IO; }
      fclose(fp);
    }
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::AREAD8; J.dirfile = pfile; J.in[0] = usew ? wfile : nullptr; J.contcheck = contcheck;
    Tool t{"AreaD8", "AreaD8", {{pfile, I16}, {wfile, F32, "weight grid does not match", SIZES, usew != 0}}, {{0, afile, F32, (double)-1.0f}}, SWEEP,
           "Number of Processes", nullptr, &J, {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input &p = g.in[0], &w = g.in[1];
      return td_aread8_outlets_host(p.as<int16_t>(), w.as<float>(), g.out<float>(0), p.nx, p.ny, p.snd(), usew ? w.fnd() : 0.f, contcheck, g.ocols, g.orows,
                                    g.nout);
    });
  });
}

// src/areadinf.cpp; a weight grid of another size is refused without a message (src/areadinf.cpp:132)
int td_area(const char* angfile, const char* scafile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, const char* wfile,
            int useOutlets, int usew, int contcheck) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::AREADINF; J.dirfile = angfile; J.in[0] = usew ? wfile : nullptr; J.contcheck = contcheck;
    Tool t{"AreaDinf", "AreaDinf", {{angfile, F32}, {wfile, F32, "weight grid does not match", SILENT, usew != 0}}, {{0, scafile, F32, (double)-1.0f}}, SWEEP,
           "Processors", nullptr, &J, {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input &a = g.in[0], &w = g.in[1];
      return td_area_outlets_host(a.as<float>(), w.as<float>(), g.out<float>(0), a.nx, a.ny, a.fnd(), usew ? w.fnd() : 0.f, a.dxc.data(), a.dyc.data(),
                                  contcheck, g.ocols, g.orows, g.nout);
    });
  });
}

// src/D8flowpathextremeup.cpp:58-285
int td_d8flowpathextremeup(const char* pfile, const char* safile, const char* ssafile, int usemax, const char* datasrc, const char* lyrname,
                           int uselyrname, int lyrno, int useOutlets, int contcheck) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::EXTREMEUP; J.dirfile = pfile; J.in[0] = safile; J.usemax = usemax; J.contcheck = contcheck;
    Tool t{"D8FlowPathExtremeUp", "D8FlowPathExtremeUp", {{pfile, I16}, {safile, F32, "value grid does not match"}}, {{0, ssafile, F32, MISSINGFLOAT}}, SWEEP,
           "Processors", nullptr, &J, {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input& p = g.in[0];
      return td_d8flowpathextremeup_host(p.as<int16_t>(), g.in[1].as<float>(), g.out<float>(0), p.nx, p.ny, p.snd(), usemax, contcheck, g.ocols, g.orows,
                                         g.nout);
    });
  });
}

// gridnet (src/gridnet.cpp:55-500)
int td_gridnet(const char* pfile, const char* plenfile, const char* tlenfile, const char* gordfile, const char* maskfile, const char* datasrc,
               const char* lyrname, int uselyrname, int lyrno, int useMask, int useOutlets, int thresh) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::GRIDNET; J.dirfile = pfile; J.in[0] = useMask == 1 ? maskfile : nullptr; J.thresh = thresh;
    Tool t{"GridNet", "GridNet", {{pfile, I16}, {maskfile, I32, "mask grid does not match", SIZES, useMask == 1}},
           {{2, gordfile, I16, -1.0}, {0, plenfile, F32, (double)-1.0f}, {1, tlenfile, F32, (double)-1.0f}}, SWEEP, "Processors", nullptr, &J,
           {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input& p = g.in[0];
      return td_gridnet_host(p.as<int16_t>(), g.in[1].as<int32_t>(), thresh, g.out<float>(0), g.out<float>(1), g.out<int16_t>(2), p.nx, p.ny, p.snd(),
                             p.dxc.data(), p.dyc.data(), g.ocols, g.orows, g.nout);
    });
  });
}

// dmarea (src/dinfdecayaccum.cpp:61-323)
int td_dmarea(const char* angfile, const char* adecfile, const char* dmfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
              const char* wfile, int useOutlets, int usew, int contcheck) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::DECAY; J.dirfile = angfile; J.in[0] = dmfile; J.in[1] = usew ? wfile : nullptr; J.contcheck = contcheck;
    Tool t{"DinfDecayAccum", "DinfDecayAccum",
           {{angfile, F32}, {dmfile, F32, "decay multiplier grid does not match"}, {wfile, F32, "weight grid does not match", SIZES, usew != 0}},
           {{0, adecfile, F32, MISSINGFLOAT}}, SWEEP, "Processors", nullptr, &J, {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input &a = g.in[0], &d = g.in[1];
      return td_dinfdecayaccum_host(a.as<float>(), d.as<float>(), g.in[2].as<float>(), g.out<float>(0), a.nx, a.ny, a.fnd(), d.fnd(), a.dxc.data(),
                                    a.dyc.data(), contcheck, g.ocols, g.orows, g.nout);
    });
  });
}

// src/DinfConcLimAccum.cpp:61-347
int td_dsllarea(const char* angfile, const char* ctptfile, const char* dmfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno,
                const char* qfile, const char* dgfile, int useOutlets, int contcheck, float cSol) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::CONCLIM; J.dirfile = angfile; J.in[0] = dmfile; J.in[1] = qfile; J.in[2] = dgfile; J.csol = cSol; J.contcheck = contcheck;
    Tool t{"DinfConcLimAccum", "DinfConcLimAccum", {{angfile, F32}, {dmfile, F32}, {dgfile, I16}, {qfile, F32}}, {{0, ctptfile, F32, MISSINGFLOAT}}, SWEEP,
           "Processors", nullptr, &J, {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input &a = g.in[0], &d = g.in[1], &q = g.in[3];
      return td_dinfconclimaccum_host(a.as<float>(), d.as<float>(), q.as<float>(), g.in[2].as<int16_t>(), g.out<float>(0), a.nx, a.ny, a.fnd(), d.fnd(),
                                      q.fnd(), cSol, a.dxc.data(), a.dyc.data(), contcheck, g.ocols, g.orows, g.nout);
    });
  });
}

// src/DinfTransLimAccum.cpp:61-394
int td_tlaccum(const char* angfile, const char* tsupfile, const char* tcfile, const char* tlafile, const char* depfile, const char* cinfile,
               const char* coutfile, const char* datasrc, const char* lyrname, int uselyrname, int lyrno, int useOutlets, int usec, int contcheck) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::TRANSLIM; J.dirfile = angfile; J.in[0] = tsupfile; J.in[1] = tcfile; J.in[2] = usec == 1 ? cinfile : nullptr; J.contcheck = contcheck;
    Tool t{"DinfTransLimAccum", "DinfTransLimAccum", {{angfile, F32}, {tsupfile, F32}, {tcfile, F32}, {cinfile, F32, "companion grid does not match", SIZES, usec == 1}},
           {{0, tlafile, F32, MISSINGFLOAT}, {1, depfile, F32, MISSINGFLOAT}, {2, coutfile, F32, MISSINGFLOAT, 0, false, usec == 1}}, SWEEP, "Processors", nullptr,
           &J, {datasrc, lyrname, uselyrname, lyrno, useOutlets}};
    return run(t, [&](const Grids& g) {
      const Input &a = g.in[0], &ts = g.in[1], &tc = g.in[2], &ci = g.in[3];
      return td_dinftranslimaccum_host(a.as<float>(), ts.as<float>(), tc.as<float>(), ci.as<float>(), g.out<float>(0), g.out<float>(1), g.out<float>(2), a.nx,
                                       a.ny, a.fnd(), ts.fnd(), tc.fnd(), usec == 1 ? ci.fnd() : 0.f, a.dxc.data(), a.dyc.data(), contcheck, g.ocols, g.orows,
                                       g.nout);
    });
  });
}

// src/Threshold.cpp:48-162; a mask of another size is refused without a message (src/Threshold.cpp:89)
int td_threshold(const char* ssafile, const char* srcfile, const char* maskfile, float thresh, int usemask) {
  return guarded([&] {
    Tool t{"Threshold", "Threshold", {{ssafile, F32}, {maskfile, F32, "mask grid does not match", SILENT, usemask == 1}}, {{0, srcfile, I16, -32768.0}}, POINT};
    return run(t, [&](const Grids& g) {
      const Input& a = g.in[0];
      return td_threshold_host(a.as<float>(), g.in[1].as<float>(), g.out<int16_t>(0), a.nx, a.ny, thresh, a.fnd());
    });
  });
}

// src/TWI.cpp:47-155; an area grid of another size is refused without a message (src/TWI.cpp:88)
int td_twigrid(const char* slopefile, const char* areafile, const char* twifile) {
  return guarded([&] {
    Tool t{"Topographic Wetness Index", "TWI", {{slopefile, F32}, {areafile, F32, "area grid does not match", SILENT}}, {{0, twifile, F32, (double)-1.0f}}, POINT};
    return run(t, [&](const Grids& g) {
      const Input &sl = g.in[0], &ar = g.in[1];
      return td_twi_host(sl.as<float>(), ar.as<float>(), g.out<float>(0), sl.nx, sl.ny, sl.fnd(), ar.fnd());
    });
  });
}

// src/SlopeArea.cpp:52-156; an area grid of another size ends in `return 1` (src/SlopeArea.cpp:89)
int td_slopearea(const char* slopefile, const char* scafile, const char* safile, const float* p) {
  return guarded([&] {
    if (!p) { td::set_error("td_slopearea: the exponents are missing"); return TD_ERR_ARG; }
    Tool t{"SlopeArea", "SlopeArea", {{slopefile, F32}, {scafile, F32, "area grid does not match", SILENT_ONE}}, {{0, safile, F32, (double)-1.0f}}, POINT};
    return run(t, [&](const Grids& g) {
      const Input& sl = g.in[0];
      return td_slopearea_host(sl.as<float>(), g.in[1].as<float>(), g.out<float>(0), sl.nx, sl.ny, p[0], p[1]);
    });
  });
}

// src/SlopeAreaRatio.cpp:49-150, the same messages as slopearea
int td_atanbgrid(const char* slopefile, const char* areafile, const char* atanbfile) {
  return guarded([&] {
    Tool t{"SlopeAreaRatio", "SlopeAreaRatio", {{slopefile, F32}, {areafile, F32, "area grid does not match", SILENT_ONE}}, {{0, atanbfile, F32, (double)-1.0f}},
           POINT};
    return run(t, [&](const Grids& g) {
      const Input &sl = g.in[0], &ar = g.in[1];
      return td_slopearearatio_host(sl.as<float>(), ar.as<float>(), g.out<float>(0), sl.nx, sl.ny, ar.fnd());
    });
  });
}

// src/PeukerDouglas.cpp:54-241: fel in, ss out (int16, nodata tag -2, georeference of fel)
int td_peukerdouglas(const char* felfile, const char* ssfile, const float* p) {
  return guarded([&] {
    if (!p) { td::set_error("td_peukerdouglas: the weights are missing"); return TD_ERR_ARG; }
    td::MgpuFlowJob J;
    J.tool = 3; J.demfile = felfile;
    for (int i = 0; i < 3; ++i) J.par[i] = p[i];
    Tool t{"PeukerDouglas", "PeukerDouglas", {{felfile, F32}}, {{0, ssfile, I16, -2.0}}, SWEEP, "Processors", &J};
    return run(t, [&](const Grids& g) {
      const Input& fel = g.in[0];
      return td_peukerdouglas_host(fel.as<float>(), g.out<int16_t>(0), fel.nx, fel.ny, fel.fnd(), p);
    });
  });
}

// src/LengthArea.cpp:51-149: plen (float) and ad8 (read as int32) in, ss out (int16, nodata -32768, georeference of ad8); an ad8 grid of
// another size ends in `return 1` there (src/LengthArea.cpp:88), TD_ERR_ARG here
int td_lengtharea(const char* plenfile, const char* ad8file, const char* ssfile, const float* p) {
  return guarded([&] {
    if (!p) { td::set_error("td_lengtharea: the coefficient and exponent are missing"); return TD_ERR_ARG; }
    Tool t{"LengthArea", "LengthArea", {{plenfile, F32}, {ad8file, I32, "ad8 grid does not match", SILENT}}, {{0, ssfile, I16, -32768.0, 1}}, POINT_COMPUTE_FIRST};
    return run(t, [&](const Grids& g) {
      const Input& pl = g.in[0];
      return td_lengtharea_host(pl.as<float>(), g.in[1].as<int32_t>(), g.out<int16_t>(0), pl.nx, pl.ny, p[0], p[1]);
    });
  });
}

// src/SlopeAveDown.cpp:59-330: fel and p in, slpd out (float32, nodata MISSINGFLOAT, the georeference of p).  The distances use fel's
// per-row cell sizes; niter uses its header cell sizes, dxA / dyA = |dxc| / |dyc| of the middle row (src/tiffIO.cpp:155).
int td_sloped(const char* pfile, const char* felfile, const char* slpdfile, double dn) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::SLOPEAVEDOWN; J.dirfile = pfile; J.in[0] = felfile; J.dn = dn;
    Tool t{"SlopeAveDown", "SlopeAveDown", {{felfile, F32}, {pfile, I16, "flow direction grid does not match"}}, {{0, slpdfile, F32, MISSINGFLOAT, 1}}, SWEEP,
           "Processors", nullptr, &J};
    double dxA = 0., dyA = 0.;
    t.opened = [&](const std::vector<Input>& in) {
      dxA = fabs(in[0].dxc[in[0].ny / 2]); dyA = fabs(in[0].dyc[in[0].ny / 2]);
      return td_slopeavedown_niter(dn, dxA, dyA, &J.niter);
    };
    return run(t, [&](const Grids& g) {
      const Input &z = g.in[0], &p = g.in[1];
      return td_slopeavedown_host(z.as<float>(), p.as<int16_t>(), g.out<float>(0), z.nx, z.ny, z.fnd(), p.snd(), z.dxc.data(), z.dyc.data(), dxA, dyA, dn);
    });
  });
}

// src/flowdircond.cpp:56-236: p (int16) and z (float) in, zfdc out (float32, the nodata value and the georeference of z: the reference
// writes zIO.getNodata(), the double of z's header).
int td_flowdircond(const char* pfile, const char* zfile, const char* zfdcfile) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::FLOWDIRCOND; J.dirfile = pfile; J.in[0] = zfile;
    Tool t{"FlowDirCond", "FlowDirCond", {{pfile, I16}, {zfile, F32, "elevation grid does not match"}}, {{0, zfdcfile, F32, 0., 1, true}}, SWEEP, "Processors",
           nullptr, &J};
    return run(t, [&](const Grids& g) {
      const Input &p = g.in[0], &z = g.in[1];
      return td_flowdircond_host(p.as<int16_t>(), z.as<float>(), g.out<float>(0), p.nx, p.ny, p.snd(), z.fnd());
    });
  });
}

// src/RetlimFlow.cpp:53-240: ang, wg and rc (float) in, qrl out (float32, nodata MISSINGFLOAT, the georeference of rc).  The shares use
// ang's per-row cell sizes.
int td_retlimro(const char* angfile, const char* wgfile, const char* rcfile, const char* qrlfile) {
  return guarded([&] {
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::RETLIMFLOW; J.dirfile = angfile; J.in[0] = wgfile; J.in[1] = rcfile;
    Tool t{"Retention limited flow accumulation", "RetlimFlow",
           {{angfile, F32}, {wgfile, F32, "weight grid does not match"}, {rcfile, F32, "retention capacity grid does not match"}},
           {{0, qrlfile, F32, MISSINGFLOAT, 2}}, SWEEP, "Processors", nullptr, &J};
    return run(t, [&](const Grids& g) {
      const Input &a = g.in[0], &w = g.in[1], &r = g.in[2];
      return td_retlimflow_host(a.as<float>(), w.as<float>(), r.as<float>(), g.out<float>(0), a.nx, a.ny, a.fnd(), w.fnd(), r.fnd(), a.dxc.data(), a.dyc.data());
    });
  });
}

// src/D8HDistToStrm.cpp:57-226 / src/D8VDistToStrm.cpp:58-240: p (int16), fel (float, vertical only) and src (int32) in, dist out
// (float32, nodata MISSINGFLOAT, the georeference of p).  The horizontal distances use p's per-row cell sizes.
static int disttostrm(bool vertical, const char* pfile, const char* felfile, const char* srcfile, const char* distfile, int thresh) {
  return guarded([&] {
    const char* name = vertical ? "D8VDistToStrm" : "D8HDistToStrm";
    td::MgpuSibJob J;
    J.tool = vertical ? td::MgpuSibJob::D8VDIST : td::MgpuSibJob::D8HDIST; J.dirfile = pfile; J.in[0] = srcfile; J.in[1] = vertical ? felfile : nullptr;
    J.thresh = thresh;
    Tool t{name, name, {{pfile, I16}, {felfile, F32, "elevation grid does not match", SIZES, vertical}, {srcfile, I32, "stream raster does not match"}},
           {{0, distfile, F32, MISSINGFLOAT}}, SWEEP, "Processors", nullptr, &J};
    return run(t, [&](const Grids& g) {
      const Input &p = g.in[0], &src = g.in[2];
      return vertical ? td_d8vdisttostrm_host(p.as<int16_t>(), g.in[1].as<float>(), src.as<int32_t>(), g.out<float>(0), p.nx, p.ny, p.snd(),
                                              (int32_t)src.r.nodata(), thresh)
                      : td_d8hdisttostrm_host(p.as<int16_t>(), src.as<int32_t>(), g.out<float>(0), p.nx, p.ny, p.snd(), (int32_t)src.r.nodata(), thresh,
                                              p.dxc.data(), p.dyc.data());
    });
  });
}
int td_distgrid(const char* pfile, const char* srcfile, const char* distfile, int thresh) {
  return disttostrm(false, pfile, nullptr, srcfile, distfile, thresh);
}
int td_d8vdistdown(const char* pfile, const char* felfile, const char* srcfile, const char* distfile, int thresh) {
  return disttostrm(true, pfile, felfile, srcfile, distfile, thresh);
}

// src/DinfDistDown.cpp:66-1398: ang (float), fel (float; v, p and s), wg (float; h, p and s with usew) and src (read as int16) in, opened
// in the reference's order (h: ang, wg, src; v: ang, fel, src; p and s: ang, fel, wg, src; slp is never opened), dd out (float32, nodata
// MISSINGFLOAT, the georeference of ang).  The shares and distances use ang's per-row cell sizes.
int td_dinfdistdown(const char* angfile, const char* felfile, const char* slpfile, const char* wfile, const char* srcfile, const char* dtsfile,
                    int statmethod, int typemethod, int usew, int concheck) {
  (void)slpfile;
  return guarded([&] {
    static const char* const banner[4] = {"DinfDistDown -h", "DinfDistDown -v", "DinfDistDown -p", "DinfDistDown -s"};
    if (typemethod < 0 || typemethod > 3 || statmethod < 0 || statmethod > 2) { td::set_error("td_dinfdistdown: bad method"); return TD_ERR_ARG; }
    const bool uf = typemethod != 0, uw = usew == 1 && typemethod != 1;
    td::MgpuSibJob J;
    J.tool = td::MgpuSibJob::DINFDISTDOWN; J.dirfile = angfile; J.in[0] = srcfile; J.in[1] = uf ? felfile : nullptr; J.in[2] = uw ? wfile : nullptr;
    J.typemethod = typemethod; J.statmethod = statmethod; J.contcheck = concheck;
    Tool t{banner[typemethod], "DinfDistDown",
           {{angfile, F32}, {felfile, F32, "elevation grid does not match", SIZES, uf}, {wfile, F32, "weight grid does not match", SIZES, uw},
            {srcfile, I16, "stream raster does not match"}},
           {{0, dtsfile, F32, MISSINGFLOAT}}, SWEEP, "Processors", nullptr, &J};
    return run(t, [&](const Grids& g) {
      const Input &a = g.in[0], &z = g.in[1], &w = g.in[2], &s = g.in[3];
      return td_dinfdistdown_host(a.as<float>(), uf ? z.as<float>() : nullptr, uw ? w.as<float>() : nullptr, s.as<int16_t>(), g.out<float>(0), a.nx, a.ny,
                                  a.fnd(), uf ? z.fnd() : 0.f, uw ? w.fnd() : 0.f, a.dxc.data(), a.dyc.data(), statmethod, typemethod, concheck);
    });
  });
}

}  // extern "C"
