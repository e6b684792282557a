// Per-device scratch owned by the library (dependency state, frontier queues,
// counters).  Everything here is device memory reused across calls.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <string>

#include "common.cuh"
#include "dinf_common.cuh"

struct td_ctx {
  // growable device buffers
  struct Buf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
      if (bytes <= cap) return cudaSuccess;
      if (p) cudaFree(p);
      p = nullptr; cap = 0;
      cudaError_t e = cudaMalloc(&p, bytes);
      if (e == cudaSuccess) cap = bytes;
      return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
  };
  Buf node;      // u16 per strip cell: static dependency node (inflow mask, dir, flags)
  Buf cnt;       // u8 per strip cell (addressed as u32 words): remaining inflow count
  Buf lev, mk;   // i32 per strip cell: Garbrecht-Martz levels / rise marks
  Buf listA, listB, listC;   // int64 cell-index lists (flat cells, BFS frontiers, ready queues)
  Buf tileflags; // fill: active-tile flags (2 x ntiles bytes)
  Buf wsched;    // warp sweep: scheduler words (head / tail / pending), one 128-byte line each
  Buf halo;      // cross-strip dependency decrements: 2 x pitch ints
  Buf theta;     // per-row atan2(dy,dx) | atan2(dx,dy) tables (doubles)
  Buf rows;      // per-row dxc | dyc (host-grid level calls)
  Buf rowfact;   // per-row constants of the flow-direction stencils (rowfact.cuh)
  Buf io[7];     // raster strips of host-grid level calls
  Buf pend;      // twi, slopearea, lengtharea: the count and list of the cells decided on the host (pointwise.cu)
  // peer mode of the sweeps (neighbour strips' buffers opened through CUDA IPC, see sweep_warp.cu)
  struct PeerInfo { void *cntw = nullptr, *tileflags = nullptr, *dctr = nullptr, *halo_in = nullptr; int qmask = 0, ntx = 0, ny = 0, th = 0, nt = 0, valid = 0, nsh = 1, qshift = 0; };
  PeerInfo peer_up, peer_down;
  void* peer_G = nullptr;                // global pending counter (rank 0's gbuf)
  bool peer_G_opened = false;
  Buf peer_halo, gbuf;
  int peer_on = 0;
  int sweep_dinf = 0;                    // which dependency state node/cnt hold
  td::PropRow prop;                      // prop() table of the strip whose theta table is loaded (uniform = 0: rows differ)
  double dx0 = 0.;                       // cell size of the strip's rows when they all have the same (prop.uniform)
  double halo_dx[2] = {0., 0.}, halo_dy[2] = {0., 0.};   // cell sizes of the neighbour strips' edge rows (row above / below; <= 0: not set, the strip's own edge rows stand in)
  static constexpr int SWEEP_KERNELS = 16;   // instantiations of the warp-per-tile sweep kernel (the table SWEEPS in sweep_warp.cu)
  int wgrid[SWEEP_KERNELS] = {0};         // persistent grid of each of them on this context's device
  static constexpr int NCTR = 40;        // device counters: [24..32] the contributing-area sweep's statistics (sweep_warp.cu WArgs::stat),
                                         // [36] slopeavedown's changed flag, [37..38] the disttostrm frontier's
                                         // appended / consumed entries (capi.cu)
  unsigned long long* d_ctr = nullptr;   // NCTR device counters
  unsigned long long* h_ctr = nullptr;   // pinned host mirror
  td_ctx();
  ~td_ctx();
};

namespace td {
void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);   // records message, returns TD_ERR_CUDA / TD_ERR_ALLOC
#define TD_CUDA(call)                                            \
  do {                                                           \
    cudaError_t e__ = (call);                                    \
    if (e__ != cudaSuccess) return ::td::cuda_fail(e__, #call);  \
  } while (0)
}  // namespace td
