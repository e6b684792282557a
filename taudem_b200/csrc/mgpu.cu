// Multi-GPU sweeps behind the executables: `TAUDEM_B200_GPUS=N aread8 ...` / `areadinf ...`, and the same for d8flowpathextremeup,
// gridnet, dinfdecayaccum, dinfconclimaccum, dinftranslimaccum, slopeavedown (whose passes follow its D8 sweep there), flowdircond,
// retlimflow, d8hdisttostrm and d8vdisttostrm (a BFS from the stream cells there): sibling_worker.  pitremove, d8flowdir,
// dinfflowdir and peukerdouglas: flow_worker.
//
// reference: the callers' contract is `mpiexec -n N aread8` (src/aread8.cpp:57,100: MPI_Init, one row strip per rank,
// src/linearpart.h:160-200 the partition, src/aread8.cpp:280-304 the border exchange + ringTerm loop).  Here the
// executable itself forks one process per GPU; every rank reads its own rows (plus one halo row either side) of the
// input rasters, runs the dependency stencil and the sweep on its device strip through the device-strip level of the
// C ABI, and stores its rows of the result into a shared mapping that the parent writes as one GeoTIFF.
//
// Two ways to get across the strip boundary:
//   peer   : the sweep kernels deliver into the neighbour GPU themselves (CUDA IPC + NVLink system-scope atomics,
//            sweep_warp.cu); the processes only exchange IPC handles through the shared mapping and meet at barriers.
//   rounds : the reference's scheme (evaluate until no cell of the strip is ready, hand the decrements and the edge rows
//            to the neighbours, repeat until nobody handed anything over), staged through the shared mapping.  Used when
//            two ranks share a device or the devices cannot reach each other; TAUDEM_B200_PEER=0/1 overrides.
// The parent never touches CUDA (a CUDA context does not survive fork()).
#include <cuda_runtime.h>
#include <sched.h>
#include <signal.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <string>
#include <vector>

#include "../../include/taudem_b200.h"
#include "mgpu.h"
#include "tiff_io.h"

namespace td {
void set_error(const std::string& msg);
void gridnet_dist_table(const double* dxc, const double* dyc, int ny, float* dist);     // capi.cu

namespace {
constexpr int MAXR = 64;
struct Shared {
  std::atomic<int> err;
  std::atomic<unsigned> bar_count, bar_gen;
  std::atomic<long long> handed[2];            // rounds mode: decrements handed over in this round (by round parity)
  double secs[MAXR];
  int rounds;
  long long flats_left;
  unsigned long long red[MAXR][8];             // allreduce_sum staging
  unsigned char handles[MAXR][320];
  int meta[MAXR][8];
  int device[MAXR], can_peer[MAXR];
  char msg[MAXR][256];
};

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// meets the other ranks; false if any rank failed (the caller bails out: nobody waits for a dead rank)
bool barrier(Shared* S, int world) {
  const unsigned gen = S->bar_gen.load();
  if (S->bar_count.fetch_add(1) + 1 == (unsigned)world) { S->bar_count.store(0); S->bar_gen.fetch_add(1); }
  else {
    for (long spins = 0; S->bar_gen.load() == gen; ++spins) {
      if (S->err.load()) return false;
      if (spins < 20000) sched_yield(); else usleep(100);
    }
  }
  return S->err.load() == 0;
}

struct Fail { std::string what; };
#define MG_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) throw Fail{std::string(#x) + ": " + cudaGetErrorString(e_)}; } while (0)
#define MG_TD(x) do { int rc_ = (x); if (rc_ != TD_OK) throw Fail{std::string(#x) + ": " + td_last_error()}; } while (0)
#define MG_BAR() do { if (!barrier(S, world)) throw Fail{"another rank failed"}; } while (0)

void partition(int total_ny, int world, int rank, int* row0, int* ny) {       // linearpart::init, src/linearpart.h:160-200
  const int n = total_ny / world;
  *row0 = rank * n;
  *ny = n + (rank == world - 1 ? total_ny % world : 0);
}

// rows [row0 - 1, row0 + ny] of a raster -> the device strip (rows 0 .. ny + 1), through a pinned buffer
void load_strip(tdio::Raster& r, tdio::DType t, void* d_strip, int nx, int pitch, int row0, int ny, int total_ny, cudaStream_t st) {
  const int eb = tdio::dtype_bytes(t);
  MG_CUDA(cudaMemsetAsync(d_strip, 0, (size_t)(ny + 2) * pitch * eb, st));
  const long first = row0 > 0 ? row0 - 1 : 0, last = std::min<long>(total_ny, (long)row0 + ny + 1);     // [first, last)
  const long blk = std::max<long>(1, (64l << 20) / ((long)nx * eb));
  void* pin[2] = {nullptr, nullptr};
  cudaEvent_t ev[2];
  for (int i = 0; i < 2; ++i) { MG_CUDA(cudaMallocHost(&pin[i], (size_t)blk * nx * eb)); MG_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming)); }
  int b = 0;
  for (long y = first; y < last; y += blk, b ^= 1) {
    const long n = std::min<long>(blk, last - y);
    MG_CUDA(cudaEventSynchronize(ev[b]));                       // the copy that used this buffer two blocks ago
    std::string err;
    if (!r.read(0, y, n, nx, pin[b], t, &err)) throw Fail{"read: " + err};
    char* dst = (char*)d_strip + (size_t)(y - row0 + 1) * pitch * eb;
    MG_CUDA(cudaMemcpy2DAsync(dst, (size_t)pitch * eb, pin[b], (size_t)nx * eb, (size_t)nx * eb, (size_t)n, cudaMemcpyHostToDevice, st));
    MG_CUDA(cudaEventRecord(ev[b], st));
  }
  MG_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < 2; ++i) { cudaFreeHost(pin[i]); cudaEventDestroy(ev[i]); }
}

struct RoundBuf {                // rounds mode: what a rank shows its neighbours (in the shared mapping, after Shared)
  static size_t bytes(int pitch) { return (size_t)pitch * (2 * sizeof(int) + 4 * sizeof(float)); }
  char* base; int pitch;
  int* halo(int rank) const { return (int*)(base + bytes(pitch) * rank); }                                  // [0,pitch): sent up, [pitch,2 pitch): sent down
  // 0 / 1 = first / last owned row of the travelling value, 2 / 3 = the same of the second one (dinftranslimaccum -cs: ctpt)
  float* row(int rank, int which) const { return (float*)(halo(rank) + 2 * pitch) + (size_t)which * pitch; }
};

// Peer mode needs every pair of neighbours on two devices that reach each other; TAUDEM_B200_PEER=0/1 overrides.
bool choose_peer(Shared* S, int rank, int world, int dev, int ndev) {
  S->device[rank] = dev;
  int can = world <= ndev ? 1 : 0;
  for (int nb = rank - 1; nb <= rank + 1 && can; nb += 2) {
    if (nb < 0 || nb >= world) continue;
    int ok = 0;
    MG_CUDA(cudaDeviceCanAccessPeer(&ok, dev, nb % ndev));
    if (!ok) can = 0;
  }
  S->can_peer[rank] = can;
  MG_BAR();
  bool peer = true;
  for (int r = 0; r < world; ++r) peer = peer && S->can_peer[r];
  if (const char* pe = getenv("TAUDEM_B200_PEER")) peer = atoi(pe) == 1;
  return peer;
}
// peer mode: every rank exports the buffers its neighbours write before anybody opens them
void peer_connect(Shared* S, int rank, int world, td_ctx* ctx, const td_strip& s, int dinf, cudaStream_t st) {
  MG_TD(td_sweep_peer_export_dev(ctx, s, dinf, S->handles[rank], S->meta[rank], st));
  MG_BAR();
  if (rank > 0) MG_TD(td_sweep_peer_connect_dev(ctx, 0, S->handles[rank - 1], S->meta[rank - 1]));
  if (rank < world - 1) MG_TD(td_sweep_peer_connect_dev(ctx, 1, S->handles[rank + 1], S->meta[rank + 1]));
  MG_TD(td_sweep_peer_connect_dev(ctx, 2, rank == 0 ? nullptr : S->handles[0], nullptr));
}
// one peer-mode sweep (after the deps call): one run per rank completes it
template <class Run>
void peer_sweep(Shared* S, int world, td_ctx* ctx, const td_strip& s, cudaStream_t st, Run&& run) {
  MG_TD(td_sweep_peer_begin_dev(ctx, s, st));
  MG_CUDA(cudaStreamSynchronize(st));
  MG_BAR();                                     // every strip is counted in the global counter before anybody can see it at zero
  run();
  MG_BAR();
}
// rounds of a downslope or upslope evaluation on row strips (after the caller has started it): run() evaluates until no cell of the
// strip is ready, writing the decrement counts it hands over into d_halo; they and the edge rows of the travelling value (val; val2 =
// a second one, or NULL) go to the neighbours; apply(dec_top, dec_bot) takes the counts received for the first / last owned row (NULL
// where there is no neighbour); repeat until nobody handed anything over.  Returns the rounds.
template <class Run, class Apply>
int exchange_rounds(Shared* S, char* extra, int rank, int world, const td_strip& s, int* d_halo, float* val, float* val2, Run&& run, Apply&& apply) {
  const int ny = s.ny;
  const RoundBuf R{extra, s.pitch};
  std::vector<int> hal(2 * (size_t)s.pitch), dec(2 * (size_t)s.pitch);
  float* vals[2] = {val, val2};
  const int nv = val2 ? 2 : 1;
  int rounds = 0;
  for (;;) {
    run();
    ++rounds;
    // what I hand over: the decrement counts and my edge rows (DistTools.share + exchange_counts, src/aread8.cpp:283-297)
    MG_CUDA(cudaMemcpy(hal.data(), d_halo, sizeof(int) * 2 * (size_t)s.pitch, cudaMemcpyDeviceToHost));
    memcpy(R.halo(rank), hal.data(), sizeof(int) * 2 * (size_t)s.pitch);
    for (int v = 0; v < nv; ++v) {
      MG_CUDA(cudaMemcpy(R.row(rank, 2 * v), vals[v] + (size_t)1 * s.pitch, sizeof(float) * s.pitch, cudaMemcpyDeviceToHost));
      MG_CUDA(cudaMemcpy(R.row(rank, 2 * v + 1), vals[v] + (size_t)ny * s.pitch, sizeof(float) * s.pitch, cudaMemcpyDeviceToHost));
    }
    long long mine = 0;
    for (int v : hal) mine += v;
    std::atomic<long long>& total = S->handed[rounds & 1];
    total.fetch_add(mine);
    MG_BAR();
    const long long all = total.load();
    std::fill(dec.begin(), dec.end(), 0);
    if (rank > 0) {                                           // what the strip above sent down, and its last row
      memcpy(dec.data(), R.halo(rank - 1) + s.pitch, sizeof(int) * s.pitch);
      for (int v = 0; v < nv; ++v) MG_CUDA(cudaMemcpy(vals[v], R.row(rank - 1, 2 * v + 1), sizeof(float) * s.pitch, cudaMemcpyHostToDevice));
    }
    if (rank < world - 1) {                                   // what the strip below sent up, and its first row
      memcpy(dec.data() + s.pitch, R.halo(rank + 1), sizeof(int) * s.pitch);
      for (int v = 0; v < nv; ++v)
        MG_CUDA(cudaMemcpy(vals[v] + (size_t)(ny + 1) * s.pitch, R.row(rank + 1, 2 * v), sizeof(float) * s.pitch, cudaMemcpyHostToDevice));
    }
    S->handed[(rounds + 1) & 1].store(0);                      // the next round's total (nobody adds to it before the barrier below)
    MG_BAR();
    if (all == 0) break;                                      // ringTerm: nobody handed anything over
    MG_CUDA(cudaMemcpy(d_halo + 2 * (size_t)s.pitch, dec.data(), sizeof(int) * 2 * (size_t)s.pitch, cudaMemcpyHostToDevice));
    apply(rank > 0 ? d_halo + 2 * (size_t)s.pitch : nullptr, rank < world - 1 ? d_halo + 3 * (size_t)s.pitch : nullptr);
  }
  return rounds;
}

// ---- the sweep tools on row strips (MgpuSibJob)
// per tool: D-infinity (ang, float) or D8 (p, int16) directions, and the types of the further inputs (MgpuSibJob::in)
struct SibTool { bool dinf; tdio::DType in[3]; };
constexpr tdio::DType F32 = tdio::DT_F32;
const SibTool sib_tools[MgpuSibJob::NTOOLS] = {
    {false, {F32, F32, F32}},            // EXTREMEUP
    {false, {tdio::DT_I32, F32, F32}},   // GRIDNET
    {true, {F32, F32, F32}},             // DECAY
    {true, {F32, F32, tdio::DT_I16}},    // CONCLIM
    {true, {F32, F32, F32}},             // TRANSLIM
    {false, {F32, F32, F32}},            // SLOPEAVEDOWN
    {false, {F32, F32, F32}},            // FLOWDIRCOND
    {true, {F32, F32, F32}},             // RETLIMFLOW
    {false, {F32, F32, F32}},            // AREAD8
    {true, {F32, F32, F32}},             // AREADINF
    {false, {tdio::DT_I32, F32, F32}},   // D8HDIST
    {false, {tdio::DT_I32, F32, F32}},   // D8VDIST
    {true, {tdio::DT_I16, F32, F32}},    // DINFDISTDOWN
};

void sibling_worker(const MgpuSibJob& J, Shared* S, char* extra, int rank, int world) {
  int ndev = 0;
  MG_CUDA(cudaGetDeviceCount(&ndev));
  if (ndev < 1) throw Fail{"no CUDA device"};
  const int dev = rank % ndev;
  MG_CUDA(cudaSetDevice(dev));
  cudaStream_t st;
  MG_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));

  const SibTool& T = sib_tools[J.tool];
  const bool dinf = T.dinf;
  tdio::Raster in;
  std::string err;
  if (!in.open(J.dirfile, &err)) throw Fail{"open " + std::string(J.dirfile) + ": " + err};
  const int nx = (int)in.width(), total_ny = (int)in.height();
  int row0, ny;
  partition(total_ny, world, rank, &row0, &ny);
  td_strip s;
  s.nx = nx; s.ny = ny; s.pitch = td_pitch_for(nx); s.has_top = rank > 0; s.has_bot = rank < world - 1;
  const size_t cells = (size_t)(ny + 2) * s.pitch;
  const tdio::DType dt = dinf ? tdio::DT_F32 : tdio::DT_I16;
  void* d_dir = nullptr;
  MG_CUDA(cudaMalloc(&d_dir, cells * tdio::dtype_bytes(dt)));
  load_strip(in, dt, d_dir, nx, s.pitch, row0, ny, total_ny, st);
  // the further inputs, each with its halo rows
  tdio::Raster rin[3];
  void* d_in[3] = {nullptr, nullptr, nullptr};
  float nd[3] = {0.f, 0.f, 0.f};
  for (int i = 0; i < 3; ++i) {
    if (!J.in[i]) continue;
    if (!rin[i].open(J.in[i], &err)) throw Fail{"open " + std::string(J.in[i]) + ": " + err};
    nd[i] = (float)rin[i].nodata();
    MG_CUDA(cudaMalloc(&d_in[i], cells * tdio::dtype_bytes(T.in[i])));
    load_strip(rin[i], T.in[i], d_in[i], nx, s.pitch, row0, ny, total_ny, st);
  }
  // the travelling value, the other outputs, gridnet's mask grid / distances / orders, the halo counts
  float *d_val = nullptr, *d_dep = nullptr, *d_co = nullptr, *d_ok = nullptr, *d_dist = nullptr; int16_t* d_g = nullptr; int* d_halo = nullptr;
  uint8_t* d_code = nullptr; float* d_state[2] = {nullptr, nullptr};                      // slopeavedown (d_code: and disttostrm)
  double* d_dx = nullptr;
  MG_CUDA(cudaMalloc(&d_val, cells * 4));
  MG_CUDA(cudaMalloc(&d_halo, sizeof(int) * 4 * (size_t)s.pitch));        // halo_out (2 pitch) + the received decrements (2 pitch)
  if (J.tool == MgpuSibJob::TRANSLIM) {
    MG_CUDA(cudaMalloc(&d_dep, cells * 4));
    if (J.in[2]) MG_CUDA(cudaMalloc(&d_co, cells * 4));
  }
  std::vector<double> dxc, dyc;
  in.cell_sizes(&dxc, &dyc);
  if (J.tool == MgpuSibJob::GRIDNET || J.tool == MgpuSibJob::SLOPEAVEDOWN || J.tool == MgpuSibJob::D8HDIST ||
      (J.tool == MgpuSibJob::DINFDISTDOWN && J.typemethod != 1)) {
    if (J.tool == MgpuSibJob::GRIDNET) {
      if (J.in[0]) MG_CUDA(cudaMalloc(&d_ok, cells * 4));
      MG_CUDA(cudaMalloc(&d_g, cells * 2));
    }
    std::vector<float> dist((size_t)ny * 8);
    gridnet_dist_table(dxc.data() + row0, dyc.data() + row0, ny, dist.data());       // this strip's own rows
    MG_CUDA(cudaMalloc(&d_dist, sizeof(float) * dist.size()));
    MG_CUDA(cudaMemcpy(d_dist, dist.data(), sizeof(float) * dist.size(), cudaMemcpyHostToDevice));
  }
  if (dinf) {
    MG_CUDA(cudaMalloc(&d_dx, sizeof(double) * 2 * (size_t)ny));
    MG_CUDA(cudaMemcpyAsync(d_dx, dxc.data() + row0, sizeof(double) * ny, cudaMemcpyHostToDevice, st));
    MG_CUDA(cudaMemcpyAsync(d_dx + ny, dyc.data() + row0, sizeof(double) * ny, cudaMemcpyHostToDevice, st));
    MG_CUDA(cudaStreamSynchronize(st));
  }
  td_ctx* ctx = td_ctx_create();
  if (!ctx) throw Fail{"td_ctx_create failed"};
  const bool peer = choose_peer(S, rank, world, dev, ndev);

  const double t0 = now();
  if (peer) peer_connect(S, rank, world, ctx, s, dinf ? 1 : 0, st);
  // the neighbour strips' edge rows keep their own cell sizes (geographic rasters: src/areadinf.cpp:199-201 getdxdyc(jn))
  if (dinf)
    td_set_halo_cell_sizes_dev(ctx, row0 > 0 ? dxc[row0 - 1] : 0., row0 > 0 ? dyc[row0 - 1] : 0., row0 + ny < total_ny ? dxc[row0 + ny] : 0.,
                               row0 + ny < total_ny ? dyc[row0 + ny] : 0.);
  int rounds = 0;
  // one sweep after its deps call: `sweep` runs the tool's *_sweep_run_dev into d_halo; val2 = a second travelling value or NULL
  auto one_sweep = [&](auto&& sweep, float* val2) {
    auto run = [&]() {
      MG_CUDA(cudaMemsetAsync(d_halo, 0, sizeof(int) * 2 * (size_t)s.pitch, st));
      sweep();
      MG_CUDA(cudaStreamSynchronize(st));
    };
    if (peer) { peer_sweep(S, world, ctx, s, st, run); rounds += 1; }
    else {
      MG_TD(td_sweep_begin_dev(ctx, s, st));
      rounds += exchange_rounds(S, extra, rank, world, s, d_halo, d_val, val2, run,
                                [&](const int* top, const int* bot) { MG_TD(td_sweep_apply_halo_dev(ctx, s, top, bot, st)); });
    }
  };
  // rows 1..ny of a strip array -> this rank's rows of an output mapping
  auto store = [&](void* out, const void* d, size_t eb) {
    MG_CUDA(cudaMemcpy2D((char*)out + (size_t)row0 * nx * eb, (size_t)nx * eb, (const char*)d + (size_t)s.pitch * eb, (size_t)s.pitch * eb, (size_t)nx * eb,
                         (size_t)ny, cudaMemcpyDeviceToHost));
  };
  const int16_t p_nd = (int16_t)in.nodata();
  const float a_nd = (float)in.nodata();
  const float* ang = (const float*)d_dir;
  const float* f0 = (const float*)d_in[0]; const float* f1 = (const float*)d_in[1]; const float* f2 = (const float*)d_in[2];
  switch (J.tool) {
    case MgpuSibJob::AREAD8:
      MG_TD(td_aread8_deps_dev(ctx, (const int16_t*)d_dir, d_val, s, p_nd, st));
      one_sweep([&]() { MG_TD(td_aread8_sweep_run_dev(ctx, f0, d_val, s, nd[0], f0 != nullptr, J.contcheck, d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::AREADINF:
      MG_TD(td_area_deps_dev(ctx, ang, d_val, s, a_nd, d_dx, d_dx + ny, st));
      one_sweep([&]() { MG_TD(td_area_sweep_run_dev(ctx, ang, f0, d_val, s, f0 != nullptr, J.contcheck, d_dx, d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::EXTREMEUP:
      MG_TD(td_d8flowpathextremeup_deps_dev(ctx, (const int16_t*)d_dir, d_val, s, p_nd, st));
      one_sweep([&]() { MG_TD(td_d8flowpathextremeup_sweep_run_dev(ctx, f0, d_val, s, J.usemax, J.contcheck, d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::GRIDNET:
      if (d_ok) MG_TD(td_gridnet_mask_dev(ctx, (const int32_t*)d_in[0], d_ok, s, J.thresh, st));
      for (int which = 0; which < 3; ++which) {        // plen, tlen, Strahler order: three sweeps in turn
        MG_TD(td_gridnet_deps_dev(ctx, (const int16_t*)d_dir, d_val, s, p_nd, st));
        one_sweep([&]() { MG_TD(td_gridnet_sweep_run_dev(ctx, which, d_ok, d_dist, d_val, s, 0, d_halo, st)); }, nullptr);
        if (which < 2) store(J.out[which], d_val, 4);
      }
      MG_TD(td_gridnet_order_dev(ctx, d_val, (const int16_t*)d_dir, d_ok, d_g, s, p_nd, 0, st));
      MG_CUDA(cudaStreamSynchronize(st));
      break;
    case MgpuSibJob::DECAY:
      MG_TD(td_dinfdecayaccum_deps_dev(ctx, ang, d_val, s, a_nd, d_dx, d_dx + ny, st));
      one_sweep([&]() { MG_TD(td_dinfdecayaccum_sweep_run_dev(ctx, ang, f0, f1, d_val, s, nd[0], J.contcheck, d_dx, d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::CONCLIM:
      MG_TD(td_dinfconclimaccum_deps_dev(ctx, ang, d_val, s, a_nd, d_dx, d_dx + ny, st));
      one_sweep([&]() { MG_TD(td_dinfconclimaccum_sweep_run_dev(ctx, ang, f0, f1, (const int16_t*)d_in[2], d_val, s, nd[0], nd[1], J.csol, J.contcheck, d_dx,
                                                                d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::FLOWDIRCOND:
      MG_TD(td_flowdircond_deps_dev(ctx, (const int16_t*)d_dir, f0, d_val, s, p_nd, st));
      one_sweep([&]() { MG_TD(td_flowdircond_sweep_run_dev(ctx, f0, d_val, s, nd[0], d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::RETLIMFLOW:
      MG_TD(td_retlimflow_deps_dev(ctx, ang, f0, f1, d_val, s, a_nd, nd[0], nd[1], d_dx, d_dx + ny, st));
      one_sweep([&]() { MG_TD(td_retlimflow_sweep_run_dev(ctx, ang, f0, f1, d_val, s, nd[0], nd[1], d_dx, d_halo, st)); }, nullptr);
      break;
    case MgpuSibJob::SLOPEAVEDOWN: {
      // the D8 sweep marks the cells the reference's queue processes; then the passes, each followed by the exchange of the state's
      // edge rows (ed->share(); dd->share(), src/SlopeAveDown.cpp:266-267) and an all-reduce of "anything changed"
      MG_TD(td_aread8_deps_dev(ctx, (const int16_t*)d_dir, d_val, s, p_nd, st));
      one_sweep([&]() { MG_TD(td_aread8_sweep_run_dev(ctx, nullptr, d_val, s, 0.f, 0, 0, d_halo, st)); }, nullptr);
      MG_CUDA(cudaMalloc(&d_code, cells));
      for (float*& b : d_state) MG_CUDA(cudaMalloc(&b, cells * 8));
      MG_TD(td_slopeavedown_init_dev(ctx, (const int16_t*)d_dir, f0, d_code, d_state[0], d_state[1], d_val, s, p_nd, nd[0], st));
      const RoundBuf R{extra, s.pitch};
      const size_t rb = (size_t)s.pitch * 8;                  // one row of the state; R.row(r, 0..1) and R.row(r, 2..3) hold two
      for (int it = 0; it < J.niter; ++it) {
        float* out = d_state[(it + 1) & 1];
        int changed = 0;
        MG_TD(td_slopeavedown_pass_dev(ctx, d_code, f0, d_state[it & 1], out, d_val, s, d_dist, J.dn, &changed, st));
        MG_CUDA(cudaMemcpy(R.row(rank, 0), (const char*)out + rb, rb, cudaMemcpyDeviceToHost));
        MG_CUDA(cudaMemcpy(R.row(rank, 2), (const char*)out + rb * (size_t)ny, rb, cudaMemcpyDeviceToHost));
        S->red[rank][0] = (unsigned long long)changed;
        MG_BAR();
        unsigned long long any = 0;
        for (int r = 0; r < world; ++r) any += S->red[r][0];
        // (on st, so that the next pass is ordered after them)
        if (rank > 0) MG_CUDA(cudaMemcpyAsync(out, R.row(rank - 1, 2), rb, cudaMemcpyHostToDevice, st));
        if (rank < world - 1) MG_CUDA(cudaMemcpyAsync((char*)out + rb * (size_t)(ny + 1), R.row(rank + 1, 0), rb, cudaMemcpyHostToDevice, st));
        MG_CUDA(cudaStreamSynchronize(st));
        ++rounds;
        MG_BAR();
        if (any == 0) break;                                  // no rank changed anything: the remaining passes would not either
      }
      break;
    }
    case MgpuSibJob::D8HDIST:
    case MgpuSibJob::D8VDIST: {
      // the reference's ring loop (src/D8HDistToStrm.cpp:158-226): BFS levels until the strip's frontier is empty, the value raster's
      // edge rows to the neighbours (fdarr->share()), and the owned edge-row cells whose receiver just got a value start the next
      // levels; until no rank added a cell (ringTerm)
      MG_CUDA(cudaMalloc(&d_code, cells));
      MG_TD(td_disttostrm_seed_dev(ctx, (const int16_t*)d_dir, (const int32_t*)d_in[0], d_val, d_code, s, J.thresh, p_nd, (int32_t)rin[0].nodata(), st));
      const RoundBuf R{extra, s.pitch};
      const size_t rb = sizeof(float) * (size_t)s.pitch;
      for (;;) {
        unsigned long long added = 0;
        MG_TD(td_disttostrm_levels_dev(ctx, J.tool == MgpuSibJob::D8VDIST, d_code, f1, d_dist, d_val, s, &added, nullptr, st));
        MG_CUDA(cudaMemcpy(R.row(rank, 0), d_val + s.pitch, rb, cudaMemcpyDeviceToHost));
        MG_CUDA(cudaMemcpy(R.row(rank, 1), d_val + (size_t)ny * s.pitch, rb, cudaMemcpyDeviceToHost));
        S->red[rank][0] = added;
        MG_BAR();
        unsigned long long any = 0;
        for (int r = 0; r < world; ++r) any += S->red[r][0];
        if (rank > 0) MG_CUDA(cudaMemcpy(d_val, R.row(rank - 1, 1), rb, cudaMemcpyHostToDevice));
        if (rank < world - 1) MG_CUDA(cudaMemcpy(d_val + (size_t)(ny + 1) * s.pitch, R.row(rank + 1, 0), rb, cudaMemcpyHostToDevice));
        ++rounds;
        MG_BAR();
        if (any == 0) break;                                  // nobody added a cell: every edge row is final
      }
      break;
    }
    case MgpuSibJob::DINFDISTDOWN: {
      // the reference's ring loop (src/DinfDistDown.cpp:243-357): levels until the strip's frontier is empty, the decrements of the
      // donors in the halo rows (neighbor->addBorders()) and the value raster's edge rows (dts->share(); two rasters in the p mode) to
      // the neighbours, the received decrements start the next levels; until nobody handed a decrement over (ringTerm)
      const bool p_mode = J.typemethod == 2;
      float* d_v = nullptr;                                   // the p mode's vertical values
      MG_CUDA(cudaMalloc(&d_code, cells));
      if (p_mode) MG_CUDA(cudaMalloc(&d_v, cells * 4));
      MG_TD(td_dinfdistdown_seed_dev(ctx, ang, (const int16_t*)d_in[0], d_val, d_v, d_code, s, a_nd, d_dx, d_dx + ny, st));
      auto run = [&]() {
        MG_CUDA(cudaMemsetAsync(d_halo, 0, sizeof(int) * 2 * (size_t)s.pitch, st));
        MG_TD(td_dinfdistdown_levels_dev(ctx, J.typemethod, J.statmethod, ang, f1, f2, d_dist, d_val, d_v, d_code, s, nd[1], nd[2], J.contcheck, d_halo,
                                         nullptr, nullptr, st));
        MG_CUDA(cudaStreamSynchronize(st));
      };
      rounds += exchange_rounds(S, extra, rank, world, s, d_halo, d_val, d_v, run,
                                [&](const int* top, const int* bot) { MG_TD(td_dinfdistdown_edge_dev(ctx, d_code, top, bot, s, st)); });
      if (p_mode) MG_TD(td_dinfdistdown_pythagoras_dev(ctx, d_val, d_v, s, st));
      MG_CUDA(cudaStreamSynchronize(st));
      cudaFree(d_v);
      break;
    }
    case MgpuSibJob::TRANSLIM:
      MG_TD(td_dinftranslimaccum_deps_dev(ctx, ang, d_val, d_dep, d_co, s, a_nd, d_dx, d_dx + ny, st));
      one_sweep([&]() { MG_TD(td_dinftranslimaccum_sweep_run_dev(ctx, ang, f0, f1, f2, d_val, d_dep, d_co, s, nd[0], nd[1], nd[2], J.contcheck, d_dx,
                                                                 d_halo, st)); }, d_co);
  }
  if (peer) td_sweep_peer_off_dev(ctx);
  S->secs[rank] = now() - t0;
  if (rank == 0) S->rounds = rounds;
  if (J.tool == MgpuSibJob::GRIDNET) store(J.out[2], d_g, 2);
  else {
    store(J.out[0], d_val, 4);
    if (d_dep) store(J.out[1], d_dep, 4);
    if (d_co) store(J.out[2], d_co, 4);
  }
  td_ctx_destroy(ctx);
  cudaFree(d_dir); cudaFree(d_val); cudaFree(d_dep); cudaFree(d_co); cudaFree(d_ok); cudaFree(d_dist); cudaFree(d_g); cudaFree(d_halo); cudaFree(d_dx);
  cudaFree(d_code); cudaFree(d_state[0]); cudaFree(d_state[1]);
  for (void* p : d_in) cudaFree(p);
}

// ---- pitremove / d8flowdir / dinfflowdir on row strips.  What the reference does with linearpart::share() and MPI_Allreduce
// (src/flood.cpp:344,401,468; src/d8.cpp:549-668) goes through the shared mapping: every rank has four row slots of 8 bytes per
// cell (its first / last owned row, its two halo rows) and a line of eight words for the sums.
struct RowSlots {
  static size_t bytes(int pitch) { return (size_t)pitch * 8 * 4; }
  char* base; int pitch;
  char* slot(int rank, int which) const { return base + bytes(pitch) * rank + (size_t)which * pitch * 8; }
};
struct StripComm {
  Shared* S; RowSlots R; int rank, world; td_strip s; cudaStream_t st;
  bool bar() const { return barrier(S, world); }
  // first / last owned row -> the halo rows of the strips above / below
  int share(void* arr, int eb) const {
    if (eb > 8) return 1;
    const size_t rb = (size_t)s.pitch * eb;
    char* a = (char*)arr;
    if (cudaMemcpyAsync(R.slot(rank, 0), a + rb, rb, cudaMemcpyDeviceToHost, st) != cudaSuccess) return 1;
    if (cudaMemcpyAsync(R.slot(rank, 1), a + rb * (size_t)s.ny, rb, cudaMemcpyDeviceToHost, st) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(st) != cudaSuccess) return 1;
    if (!bar()) return 1;
    if (rank > 0 && cudaMemcpyAsync(a, R.slot(rank - 1, 1), rb, cudaMemcpyHostToDevice, st) != cudaSuccess) return 1;
    if (rank < world - 1 && cudaMemcpyAsync(a + rb * (size_t)(s.ny + 1), R.slot(rank + 1, 0), rb, cudaMemcpyHostToDevice, st) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(st) != cudaSuccess) return 1;
    return bar() ? 0 : 1;
  }
  // the reverse: what the neighbours hold in their halo rows for my first / last row
  int collect(const void* arr, int eb, void* recv_top, void* recv_bot) const {
    if (eb > 8) return 1;
    const size_t rb = (size_t)s.pitch * eb;
    const char* a = (const char*)arr;
    if (cudaMemcpyAsync(R.slot(rank, 2), a, rb, cudaMemcpyDeviceToHost, st) != cudaSuccess) return 1;
    if (cudaMemcpyAsync(R.slot(rank, 3), a + rb * (size_t)(s.ny + 1), rb, cudaMemcpyDeviceToHost, st) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(st) != cudaSuccess) return 1;
    if (!bar()) return 1;
    if (rank > 0 && recv_top && cudaMemcpyAsync(recv_top, R.slot(rank - 1, 3), rb, cudaMemcpyHostToDevice, st) != cudaSuccess) return 1;
    if (rank < world - 1 && recv_bot && cudaMemcpyAsync(recv_bot, R.slot(rank + 1, 2), rb, cudaMemcpyHostToDevice, st) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(st) != cudaSuccess) return 1;
    return bar() ? 0 : 1;
  }
  int allreduce_sum(unsigned long long* v, int n) const {
    if (n > 8) return 1;
    for (int i = 0; i < n; ++i) S->red[rank][i] = v[i];
    if (!bar()) return 1;
    for (int i = 0; i < n; ++i) { unsigned long long t = 0; for (int r = 0; r < world; ++r) t += S->red[r][i]; v[i] = t; }
    return bar() ? 0 : 1;
  }
};
int cb_share(void* u, void* arr, int eb) { return ((const StripComm*)u)->share(arr, eb); }
int cb_collect(void* u, const void* arr, int eb, void* rt, void* rb) { return ((const StripComm*)u)->collect(arr, eb, rt, rb); }
int cb_allreduce(void* u, unsigned long long* v, int n) { return ((const StripComm*)u)->allreduce_sum(v, n); }

void flow_worker(const MgpuFlowJob& J, Shared* S, char* extra, int rank, int world) {
  int ndev = 0;
  MG_CUDA(cudaGetDeviceCount(&ndev));
  if (ndev < 1) throw Fail{"no CUDA device"};
  MG_CUDA(cudaSetDevice(rank % ndev));
  cudaStream_t st;
  MG_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  tdio::Raster in, mk;
  std::string err;
  if (!in.open(J.demfile, &err)) throw Fail{"open " + std::string(J.demfile) + ": " + err};
  const int nx = (int)in.width(), total_ny = (int)in.height();
  if (J.tool == 0 && J.use_mask && !mk.open(J.maskfile, &err)) throw Fail{"open " + std::string(J.maskfile) + ": " + err};
  int row0, ny;
  partition(total_ny, world, rank, &row0, &ny);
  td_strip s;
  s.nx = nx; s.ny = ny; s.pitch = td_pitch_for(nx); s.has_top = rank > 0; s.has_bot = rank < world - 1;
  const size_t cells = (size_t)(ny + 2) * s.pitch;
  float *d_z = nullptr, *d_f = nullptr, *d_slp = nullptr; void* d_dir = nullptr; int16_t* d_mask = nullptr; double* d_dx = nullptr;
  MG_CUDA(cudaMalloc(&d_z, cells * 4));
  load_strip(in, tdio::DT_F32, d_z, nx, s.pitch, row0, ny, total_ny, st);
  td_ctx* ctx = td_ctx_create();
  if (!ctx) throw Fail{"td_ctx_create failed"};
  const StripComm C{S, RowSlots{extra, s.pitch}, rank, world, s, st};
  td_strip_comm comm;
  comm.user = (void*)&C; comm.share = cb_share; comm.collect = cb_collect; comm.allreduce_sum = cb_allreduce;
  MG_BAR();
  const double t0 = now();
  int rounds = 0;
  long long left = 0;
  if (J.tool == 0) {
    // flood(): local relaxation to convergence, fresh halo rows, repeat until no strip moved (src/flood.cpp:344-479)
    if (J.use_mask) { MG_CUDA(cudaMalloc(&d_mask, cells * 2)); load_strip(mk, tdio::DT_I16, d_mask, nx, s.pitch, row0, ny, total_ny, st); }
    MG_CUDA(cudaMalloc(&d_f, cells * 4));
    MG_CUDA(cudaMemsetAsync(d_f, 0, cells * 4, st));
    MG_TD(td_flood_init_dev(ctx, d_z, d_mask, d_f, s, (float)in.nodata(), J.four, st));
    for (bool first = true;; first = false) {
      MG_CUDA(cudaStreamSynchronize(st));
      if (C.share(d_f, 4)) throw Fail{"row exchange failed"};
      int moved = 0;
      if (first) MG_TD(td_flood_relax_dev(ctx, d_z, d_f, s, J.four, &moved, st));
      else MG_TD(td_flood_relax_edges_dev(ctx, d_z, d_f, s, J.four, &moved, st));
      ++rounds;
      unsigned long long any = moved ? 1ull : 0ull;
      if (C.allreduce_sum(&any, 1)) throw Fail{"all-reduce failed"};
      if (any == 0) break;
    }
    MG_CUDA(cudaMemcpy2D((float*)J.out[0] + (size_t)row0 * nx, (size_t)nx * 4, d_f + s.pitch, (size_t)s.pitch * 4, (size_t)nx * 4, (size_t)ny, cudaMemcpyDeviceToHost));
  } else if (J.tool == 3) {
    // peukerdouglas: smoothing on the raw halo rows, the smoothed edge rows to the neighbours (src/PeukerDouglas.cpp:165), marks
    MG_CUDA(cudaMalloc(&d_f, cells * 4));
    MG_CUDA(cudaMalloc(&d_dir, cells * 2));
    MG_CUDA(cudaMemsetAsync(d_f, 0, cells * 4, st));
    MG_TD(td_peukerdouglas_smooth_dev(ctx, d_z, d_f, s, (float)in.nodata(), J.par, st));
    MG_CUDA(cudaStreamSynchronize(st));
    if (C.share(d_f, 4)) throw Fail{"row exchange failed"};
    MG_TD(td_peukerdouglas_mark_dev(ctx, d_f, (int16_t*)d_dir, s, (float)in.nodata(), st));
    MG_CUDA(cudaStreamSynchronize(st));
    rounds = 1;
    MG_CUDA(cudaMemcpy2D((int16_t*)J.out[0] + (size_t)row0 * nx, (size_t)nx * 2, (int16_t*)d_dir + s.pitch, (size_t)s.pitch * 2, (size_t)nx * 2, (size_t)ny,
                         cudaMemcpyDeviceToHost));
  } else {
    const bool dinf = J.tool == 2;
    std::vector<double> dxc, dyc;
    in.cell_sizes(&dxc, &dyc);
    MG_CUDA(cudaMalloc(&d_dx, sizeof(double) * 2 * (size_t)ny));
    MG_CUDA(cudaMemcpyAsync(d_dx, dxc.data() + row0, sizeof(double) * ny, cudaMemcpyHostToDevice, st));
    MG_CUDA(cudaMemcpyAsync(d_dx + ny, dyc.data() + row0, sizeof(double) * ny, cudaMemcpyHostToDevice, st));
    const size_t eb = dinf ? 4 : 2;
    MG_CUDA(cudaMalloc(&d_dir, cells * eb));
    MG_CUDA(cudaMalloc(&d_slp, cells * 4));
    MG_CUDA(cudaMemsetAsync(d_dir, 0, cells * eb, st));
    MG_CUDA(cudaMemsetAsync(d_slp, 0, cells * 4, st));
    MG_CUDA(cudaStreamSynchronize(st));
    long long nflat = 0;
    if (dinf) MG_TD(td_dinf_slopes_dev(ctx, d_z, (float*)d_dir, d_slp, s, (float)in.nodata(), d_dx, d_dx + ny, &nflat, st));
    else MG_TD(td_d8_slopes_dev(ctx, d_z, (int16_t*)d_dir, d_slp, s, (float)in.nodata(), d_dx, d_dx + ny, &nflat, st));
    MG_CUDA(cudaStreamSynchronize(st));
    unsigned long long total = (unsigned long long)nflat;
    if (C.allreduce_sum(&total, 1)) throw Fail{"all-reduce failed"};
    if (total) {
      // Garbrecht-Martz on the strips: the halo rows of the directions first, then the BFS passes with their exchanges
      if (C.share(d_dir, (int)eb)) throw Fail{"row exchange failed"};
      if (dinf) MG_TD(td_dinf_flats_strip_dev(ctx, d_z, (float*)d_dir, s, d_dx, d_dx + ny, &left, &comm, st));
      else MG_TD(td_d8_flats_strip_dev(ctx, d_z, (int16_t*)d_dir, s, d_dx, d_dx + ny, &left, &comm, st));
      MG_CUDA(cudaStreamSynchronize(st));
    }
    MG_CUDA(cudaMemcpy2D((char*)J.out[0] + (size_t)row0 * nx * eb, (size_t)nx * eb, (char*)d_dir + (size_t)s.pitch * eb, (size_t)s.pitch * eb, (size_t)nx * eb, (size_t)ny,
                         cudaMemcpyDeviceToHost));
    MG_CUDA(cudaMemcpy2D((float*)J.out[1] + (size_t)row0 * nx, (size_t)nx * 4, d_slp + s.pitch, (size_t)s.pitch * 4, (size_t)nx * 4, (size_t)ny, cudaMemcpyDeviceToHost));
  }
  S->secs[rank] = now() - t0;
  if (rank == 0) { S->rounds = rounds; S->flats_left = left; }
  td_ctx_destroy(ctx);
  cudaFree(d_z); cudaFree(d_f); cudaFree(d_slp); cudaFree(d_dir); cudaFree(d_mask); cudaFree(d_dx);
}
}  // namespace

void* mgpu_alloc_shared(size_t bytes) {
  void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
  return p == MAP_FAILED ? nullptr : p;
}
void mgpu_free_shared(void* p, size_t bytes) { if (p) munmap(p, bytes); }

int mgpu_world() {
  const char* e = getenv("TAUDEM_B200_GPUS");
  const int n = e ? atoi(e) : 1;
  return n < 1 ? 1 : (n > MAXR ? MAXR : n);
}

namespace {
// forks `world` ranks over a shared control block (+ extra bytes), waits for them, collects the timings
template <class Fn>
int run_ranks(const char* who, int world, size_t extra_bytes, Fn&& rank_fn, double* compute_seconds, int* rounds, long long* flats_left) {
  const size_t bytes = sizeof(Shared) + extra_bytes;
  char* mem = (char*)mgpu_alloc_shared(bytes);
  if (!mem) { set_error(std::string(who) + ": cannot map the shared control block"); return TD_ERR_IO; }
  Shared* S = new (mem) Shared();
  S->err.store(0); S->bar_count.store(0); S->bar_gen.store(0); S->handed[0].store(0); S->handed[1].store(0);
  fflush(stdout); fflush(stderr);
  std::vector<pid_t> pids(world, (pid_t)-1);
  for (int r = 0; r < world; ++r) {
    const pid_t pid = fork();
    if (pid < 0) { S->err.store(1); break; }
    if (pid == 0) {
      int code = 0;
      try { rank_fn(S, mem + sizeof(Shared), r); }
      catch (const Fail& f) { snprintf(S->msg[r], sizeof(S->msg[r]), "%s", f.what.c_str()); code = 1; }
      catch (const std::exception& e) { snprintf(S->msg[r], sizeof(S->msg[r]), "exception: %s", e.what()); code = 1; }
      if (code) S->err.store(1);
      fflush(stdout); fflush(stderr);
      _exit(code);                                  // no atexit handlers of the parent's image in the child
    }
    pids[r] = pid;
  }
  // the parent only waits: a rank that dies takes the others with it (they see err at their next barrier; ranks that are
  // stuck in a kernel waiting for the dead one are killed after a grace period)
  int left = 0, bad = 0;
  for (pid_t p : pids) if (p > 0) ++left;
  double t_err = 0.;
  while (left > 0) {
    bool any = false;
    for (int r = 0; r < world; ++r) {
      if (pids[r] <= 0) continue;
      int status = 0;
      const pid_t w = waitpid(pids[r], &status, WNOHANG);
      if (w == pids[r]) {
        any = true; pids[r] = -1; --left;
        if (!WIFEXITED(status) || WEXITSTATUS(status) != 0) {
          ++bad; S->err.store(1);
          if (!S->msg[r][0]) snprintf(S->msg[r], sizeof(S->msg[r]), "rank ended abnormally (status 0x%x)", status);
        }
      }
    }
    if (S->err.load()) {
      if (t_err == 0.) t_err = now();
      else if (now() - t_err > 20.) { for (pid_t p : pids) if (p > 0) kill(p, SIGKILL); }
    }
    if (!any) usleep(2000);
  }
  int rc = TD_OK;
  if (bad || S->err.load()) {
    std::string m = "multi-GPU run failed:";
    for (int r = 0; r < world; ++r) if (S->msg[r][0] && strcmp(S->msg[r], "another rank failed") != 0) m += " [rank " + std::to_string(r) + "] " + S->msg[r];
    set_error(m);
    rc = TD_ERR_CUDA;
  } else {
    double mx = 0.;
    for (int r = 0; r < world; ++r) mx = std::max(mx, S->secs[r]);
    if (compute_seconds) *compute_seconds = mx;
    if (rounds) *rounds = S->rounds;
    if (flats_left) *flats_left = S->flats_left;
  }
  mgpu_free_shared(mem, bytes);
  return rc;
}
}  // namespace

int mgpu_sibling(const MgpuSibJob& J, int world, double* compute_seconds, int* rounds) {
  if (world < 2 || world > MAXR) { set_error("mgpu_sibling: between 2 and 64 ranks"); return TD_ERR_ARG; }
  if (J.ny < world) { set_error("mgpu_sibling: fewer rows than ranks"); return TD_ERR_ARG; }
  if (J.tool < 0 || J.tool >= MgpuSibJob::NTOOLS || !J.out[0]) { set_error("mgpu_sibling: bad job"); return TD_ERR_ARG; }
  const int pitch = td_pitch_for(J.nx);
  return run_ranks("mgpu_sibling", world, RoundBuf::bytes(pitch) * (size_t)world,
                   [&](Shared* S, char* extra, int r) { sibling_worker(J, S, extra, r, world); }, compute_seconds, rounds, nullptr);
}

int mgpu_flow(const MgpuFlowJob& J, int world, double* compute_seconds, int* rounds, long long* flats_left) {
  if (world < 2 || world > MAXR) { set_error("mgpu_flow: between 2 and 64 ranks"); return TD_ERR_ARG; }
  if (J.ny < world) { set_error("mgpu_flow: fewer rows than ranks"); return TD_ERR_ARG; }
  if (J.tool < 0 || J.tool > 3 || !J.out[0] || ((J.tool == 1 || J.tool == 2) && !J.out[1])) { set_error("mgpu_flow: bad job"); return TD_ERR_ARG; }
  const int pitch = td_pitch_for(J.nx);
  return run_ranks("mgpu_flow", world, RowSlots::bytes(pitch) * (size_t)world,
                   [&](Shared* S, char* extra, int r) { flow_worker(J, S, extra, r, world); }, compute_seconds, rounds, flats_left);
}

}  // namespace td
