// Multi-GPU sweeps and flow directions behind the file-level entry points (mgpu.cu): one forked process per GPU.
#pragma once
#include <stddef.h>

namespace td {
// pitremove, the flow directions and peukerdouglas on row strips: tool 0 = pitremove (out[0] = fel), 1 = d8flowdir (out[0] = p int16,
// out[1] = sd8), 2 = dinfflowdir (out[0] = ang, out[1] = slp), 3 = peukerdouglas (out[0] = ss int16); the rasters live in mappings from
// mgpu_alloc_shared
struct MgpuFlowJob {
  int tool = 0;
  const char* demfile = nullptr;
  const char* maskfile = nullptr;   // pitremove: depression mask (use_mask)
  int use_mask = 0, four = 0;
  float par[3] = {0.4f, 0.1f, 0.05f};   // peukerdouglas: smoothing weights
  int nx = 0, ny = 0;
  void* out[2] = {nullptr, nullptr};
};
// the sweep tools on row strips; in[] = the further inputs (NULL = not used) and out[] = the outputs (mappings from
// mgpu_alloc_shared, nx * ny cells of the output's type) of each tool:
//   EXTREMEUP  d8flowpathextremeup  in: sa                 out: ssa
//   GRIDNET    gridnet              in: mask (int32)       out: plen, tlen, gord (int16)
//   DECAY      dinfdecayaccum       in: dm, w              out: dsca
//   CONCLIM    dinfconclimaccum     in: dm, q, dg (int16)  out: ctpt
//   TRANSLIM   dinftranslimaccum    in: tsup, tc, cs       out: tla, tdep, ctpt (with cs)
//   SLOPEAVEDOWN  slopeavedown      in: fel                out: slpd (the D8 sweep of p, then niter passes at dn)
//   FLOWDIRCOND   flowdircond       in: z                  out: zfdc
//   RETLIMFLOW    retlimflow        in: wg, rc             out: qrl
//   AREAD8        aread8            in: w (or NULL)        out: ad8
//   AREADINF      areadinf          in: w (or NULL)        out: sca
//   D8HDIST       d8hdisttostrm     in: src (int32)        out: dist (thresh)
//   D8VDIST       d8vdisttostrm     in: src (int32), fel   out: dist (thresh)
//   DINFDISTDOWN  dinfdistdown      in: src (int16), fel (or NULL), w (or NULL)   out: dd (typemethod, statmethod, contcheck)
struct MgpuSibJob {
  enum { EXTREMEUP = 0, GRIDNET, DECAY, CONCLIM, TRANSLIM, SLOPEAVEDOWN, FLOWDIRCOND, RETLIMFLOW, AREAD8, AREADINF, D8HDIST, D8VDIST, DINFDISTDOWN,
         NTOOLS };
  int tool = EXTREMEUP;
  const char* dirfile = nullptr;              // p (D8 tools) or ang
  const char* in[3] = {nullptr, nullptr, nullptr};
  int usemax = 1, contcheck = 1, thresh = 0;   // thresh: gridnet, d8hdisttostrm, d8vdisttostrm
  float csol = 0.f;
  double dn = 0.; int niter = 0;              // slopeavedown
  int typemethod = 0, statmethod = 0;         // dinfdistdown
  int nx = 0, ny = 0;
  void* out[3] = {nullptr, nullptr, nullptr};
};
int mgpu_world();                                // TAUDEM_B200_GPUS (1 = the single-GPU path)
void* mgpu_alloc_shared(size_t bytes);             // anonymous shared mapping (visible to the forked ranks)
void mgpu_free_shared(void* p, size_t bytes);
// runs the job on `world` ranks; compute_seconds = the slowest rank's time from the dependency stencil to the end of the sweep;
// rounds: summed over gridnet's three sweeps, 1 per sweep in peer mode
int mgpu_sibling(const MgpuSibJob& job, int world, double* compute_seconds, int* rounds);
// rounds = relaxation / exchange rounds of pitremove, 0 for the flow directions; flats_left = unresolved flat cells of the whole grid
int mgpu_flow(const MgpuFlowJob& job, int world, double* compute_seconds, int* rounds, long long* flats_left);
}  // namespace td
